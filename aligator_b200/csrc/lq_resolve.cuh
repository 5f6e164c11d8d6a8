// lq_resolve.cuh -- the vector half of the Riccati recursion, for many right-hand sides per instance
// (ab2_gar_resolve, include/aligator_b200/gar.h).  Plain C++ apart from the execution context, so that the host
// emulation (tests/emu/resolve_emu.cpp) compiles the same program and runs it on emulated lanes.
//
// Given the factorisation the last backward left in HBM -- the gains FB = [K; Z; Ahat] and the cost-to-go Hessians
// Vxx -- and new vectors h = (q_t, r_t, d_t, f_t, q_N, d_N, g0), one work item (instance b, right-hand sides
// [j0, j0 + R)) computes z = -K^-1 h, the solution of the same LQ problem with its vectors replaced by h:
//   terminal   z_N = d_N / mu,   vx_N = q_N + C_N^T z_N
//   stage t    V' = Vxx_{t+1},  v+ = vx_{t+1} + V' f_t,  rhat = r_t + B^T v+,
//              [k; z] = -KKT^-1 [rhat; d_t] with KKT = [[R + B^T V' B, D^T], [D, -mu I]] (Bunch-Kaufman, here),
//              a = f_t + B k,  vx_t = (qhat + Shat k) + C^T z,  qhat = q_t + A^T v+,  Shat k = S k + A^T V' B k
//   initial    [x_0; lam_0] = -[[Vxx_0, G0^T], [G0, 0]]^-1 [vx_0; g0]
//   forward    u = k + K x,  v = z + Z x,  x+ = a + Ahat x,  lam_{t+1} = vx_{t+1} + Vxx_{t+1} x+,
//              v_N = z_N + Z_N x_N.
// vx_t is formed in the reference's order from the solved k and z.  The shorter form q_t + Ahat^T v+ + K^T r_t +
// Z^T d_t (equal in exact arithmetic, and free of A, S and C) multiplies the rounding error of the stored gains by
// |v+|, which grows like 1/mu with terminal constraints: it misses the extended-precision bar by four orders of
// magnitude at mu = 1e-8 (tests/test_resolve_oracle.py).
//
// Every saddle-point matrix is read from its lower triangle (V' and Vxx_0 included), as the sweep's Bunch-Kaufman
// factorisations read theirs.  The backward pass parks its per-knot vectors in the caller's output arrays: k in us[t],
// z in vs[t], a in xs[t+1], vx_{t+1} in lams[t]; the forward pass reads each back and overwrites it with the solution.
// So the call needs no scratch memory: nu + nc + 2 nx doubles per knot and right-hand side are written twice and
// read once.
//
// Work split: one item per (instance, chunk of right-hand sides), run by `nl` lanes that synchronise with ctx.sync()
// (one warp on the device).  The knot's matrices are staged once per item and shared by the chunk; each entry of a
// vector result is computed by one lane in a fixed order, so a right-hand side's result does not depend on the chunk
// it shares or on the lane count.
#pragma once

#if defined(__CUDACC__)
#define AB2_RS_HD __host__ __device__ __forceinline__
#else
#define AB2_RS_HD inline
#endif

#include <math.h>

#include "lq_record.cuh"
#include "vxx_layout.h"

namespace ab2 {

struct ResolveArgs {
  int batch, N, nx, nu, nc, nct, nc0, srec, trec, stage_head;
  int nrhs, chunk;              // right-hand sides, and how many one item holds on chip
  const double *stage, *term, *G0;
  const double *fb, *fbT;       // FB [batch][N][(nu+nc+nx)*nx] (row-major), FBT [batch][nct*nx]
  const double *Vxx, *Vxx0;     // Vxx0 != null: packed layout of vxx_layout.h; else [batch][N+1][nx*nx]
  double mueq;
  const double *mueq_b;         // per-instance mu, or null
  const double *q, *r, *d, *dN, *g0, *f;           // [nrhs][batch][...]; null = zero
  double *xs, *us, *vs, *vsT, *lam0, *lams;        // [nrhs][batch][...]
};

// doubles of shared memory one item uses
AB2_RS_HD int resolve_nkkt(int nu, int nc, int nx, int nc0) {
  const int n = nu + nc, n0 = nx + nc0;
  return n > n0 ? n : n0;
}
// The matrix region holds, in turn, a stage knot's V', [A | S | C] (backward) or FB rows (forward, the same nr * nx
// doubles), B, V'B, KKT matrix and pivots, and the initial saddle matrix and its pivots, which are formed when the stage
// buffers are dead.
AB2_RS_HD int resolve_mat_doubles(int nx, int nu, int nc, int nc0) {
  const int nr = nu + nc + nx, n = nu + nc, n0 = nx + nc0;
  const int stage = nx * nx + nr * nx + 2 * nx * nu + n * n + n;
  const int init = n0 * n0 + n0;
  return stage > init ? stage : init;
}
AB2_RS_HD int resolve_item_doubles(int nx, int nu, int nc, int nc0, int chunk) {
  const int per = 4 * nx + resolve_nkkt(nu, nc, nx, nc0); // x, x+, v+, vx, solve vector
  return ((resolve_mat_doubles(nx, nu, nc, nc0) + chunk * per) + 1) & ~1;
}

namespace rs {

// entry (i, j), i >= j, of knot `slot`'s Vxx
AB2_RS_HD double vxx_lower(const ResolveArgs &a, long b, int slot, int i, int j) {
  const int nx = a.nx;
  if (a.Vxx0) {
    if (vxx_slot_is_full(slot))
      return a.Vxx0[b * nx * nx + i + (long)j * nx];
    return a.Vxx[(b * (a.N + 1) + slot) * vxx_packed_doubles(nx) + vxx_packed_index(nx, i, j)];
  }
  return a.Vxx[(b * (a.N + 1) + slot) * nx * nx + i + (long)j * nx];
}

// V (nx x nx, column-major, symmetric) <- Vxx of `slot` from its lower triangle
template <class Ctx>
AB2_RS_HD void load_v(const ResolveArgs &a, const Ctx &ctx, long b, int slot, double *V) {
  const int nx = a.nx;
  for (int e = ctx.lane; e < nx * nx; e += ctx.nl) {
    const int i = e % nx, j = e / nx;
    V[e] = i >= j ? vxx_lower(a, b, slot, i, j) : vxx_lower(a, b, slot, j, i);
  }
}

// Bunch-Kaufman factorisation P A P^T = L D L^T of the n x n matrix whose LOWER triangle is in A (column-major,
// leading dimension n), in place (LAPACK dsytf2, lower): L below the diagonal, D on the diagonal and first
// subdiagonal; piv[k] = k' >= 0 for a 1x1 pivot interchanged with k', piv[k] = piv[k+1] = -(k'+1) for a 2x2 pivot
// whose second row was interchanged with k'.  Every lane takes the same pivot decisions; the updates are split.
template <class Ctx>
AB2_RS_HD void bk_factor(const Ctx &ctx, double *A, double *piv, int n) {
  const double alpha = (1.0 + sqrt(17.0)) / 8.0;
  int k = 0;
  while (k < n) {
    int kstep = 1, kp = k;
    const double absakk = fabs(A[k + k * n]);
    int imax = k;
    double colmax = 0.0;
    for (int i = k + 1; i < n; ++i)
      if (fabs(A[i + k * n]) > colmax) {
        colmax = fabs(A[i + k * n]);
        imax = i;
      }
    const bool zero = (absakk > colmax ? absakk : colmax) == 0.0;
    if (!zero && absakk < alpha * colmax) {
      double rowmax = 0.0;
      for (int j = k; j < imax; ++j)
        rowmax = fabs(A[imax + j * n]) > rowmax ? fabs(A[imax + j * n]) : rowmax;
      for (int j = imax + 1; j < n; ++j)
        rowmax = fabs(A[j + imax * n]) > rowmax ? fabs(A[j + imax * n]) : rowmax;
      if (absakk >= alpha * colmax * (colmax / rowmax)) {
        kp = k;
      } else if (fabs(A[imax + imax * n]) >= alpha * rowmax) {
        kp = imax;
      } else {
        kp = imax;
        kstep = 2;
      }
    }
    ctx.sync(); // every lane has read what the interchange moves
    const int kk = k + kstep - 1;
    if (kp != kk) { // interchange rows and columns kk and kp of the trailing lower triangle
      for (int i = kp + 1 + ctx.lane; i < n; i += ctx.nl) {
        const double t = A[i + kk * n];
        A[i + kk * n] = A[i + kp * n];
        A[i + kp * n] = t;
      }
      for (int j = kk + 1 + ctx.lane; j < kp; j += ctx.nl) {
        const double t = A[j + kk * n];
        A[j + kk * n] = A[kp + j * n];
        A[kp + j * n] = t;
      }
      if (ctx.lane == 0) {
        const double t = A[kk + kk * n];
        A[kk + kk * n] = A[kp + kp * n];
        A[kp + kp * n] = t;
        if (kstep == 2) {
          const double u = A[k + 1 + k * n];
          A[k + 1 + k * n] = A[kp + k * n];
          A[kp + k * n] = u;
        }
      }
    }
    ctx.sync();
    const int m = n - k - kstep; // trailing size
    if (kstep == 1) {
      if (!zero) {
        const double d11 = 1.0 / A[k + k * n];
        for (int e = ctx.lane; e < m * m; e += ctx.nl) {
          const int i = k + 1 + e % m, j = k + 1 + e / m;
          if (i >= j)
            A[i + j * n] -= d11 * A[i + k * n] * A[j + k * n];
        }
        ctx.sync();
        for (int i = k + 1 + ctx.lane; i < n; i += ctx.nl)
          A[i + k * n] *= d11;
      }
      if (ctx.lane == 0)
        piv[k] = kp;
    } else {
      if (m > 0) {
        double d21 = A[k + 1 + k * n];
        const double d11 = A[k + 1 + (k + 1) * n] / d21, d22 = A[k + k * n] / d21;
        const double t = 1.0 / (d11 * d22 - 1.0);
        d21 = t / d21;
        for (int e = ctx.lane; e < m * m; e += ctx.nl) {
          const int i = k + 2 + e % m, j = k + 2 + e / m;
          if (i >= j) {
            const double wk = d21 * (d11 * A[j + k * n] - A[j + (k + 1) * n]);
            const double wkp1 = d21 * (d22 * A[j + (k + 1) * n] - A[j + k * n]);
            A[i + j * n] -= A[i + k * n] * wk + A[i + (k + 1) * n] * wkp1;
          }
        }
        ctx.sync();
        for (int j = k + 2 + ctx.lane; j < n; j += ctx.nl) {
          const double wk = d21 * (d11 * A[j + k * n] - A[j + (k + 1) * n]);
          const double wkp1 = d21 * (d22 * A[j + (k + 1) * n] - A[j + k * n]);
          A[j + k * n] = wk;
          A[j + (k + 1) * n] = wkp1;
        }
      }
      if (ctx.lane == 0)
        piv[k] = piv[k + 1] = -(double)(kp + 1);
    }
    ctx.sync();
    k += kstep;
  }
}

// x <- A^-1 x with the factorisation of bk_factor (LAPACK dsytrs, lower); one lane, one right-hand side
AB2_RS_HD void bk_solve(const double *A, const double *piv, int n, double *x) {
  int k = 0;
  while (k < n) { // L D y = P x
    if (piv[k] >= 0.0) {
      const int kp = (int)piv[k];
      if (kp != k) {
        const double t = x[k];
        x[k] = x[kp];
        x[kp] = t;
      }
      for (int i = k + 1; i < n; ++i)
        x[i] -= A[i + k * n] * x[k];
      x[k] /= A[k + k * n];
      k += 1;
    } else {
      const int kp = -(int)piv[k] - 1;
      if (kp != k + 1) {
        const double t = x[k + 1];
        x[k + 1] = x[kp];
        x[kp] = t;
      }
      for (int i = k + 2; i < n; ++i)
        x[i] -= A[i + k * n] * x[k] + A[i + (k + 1) * n] * x[k + 1];
      const double akm1k = A[k + 1 + k * n];
      const double akm1 = A[k + k * n] / akm1k, ak = A[k + 1 + (k + 1) * n] / akm1k;
      const double denom = akm1 * ak - 1.0;
      const double bkm1 = x[k] / akm1k, bk = x[k + 1] / akm1k;
      x[k] = (ak * bkm1 - bk) / denom;
      x[k + 1] = (akm1 * bk - bkm1) / denom;
      k += 2;
    }
  }
  k = n - 1;
  while (k >= 0) { // L^T P x = y
    double s = x[k];
    for (int i = k + 1; i < n; ++i)
      s -= A[i + k * n] * x[i];
    x[k] = s;
    if (piv[k] >= 0.0) {
      const int kp = (int)piv[k];
      if (kp != k) {
        const double t = x[k];
        x[k] = x[kp];
        x[kp] = t;
      }
      k -= 1;
    } else {
      double s1 = x[k - 1];
      for (int i = k + 1; i < n; ++i)
        s1 -= A[i + (k - 1) * n] * x[i];
      x[k - 1] = s1;
      const int kp = -(int)piv[k] - 1;
      if (kp != k) {
        const double t = x[k];
        x[k] = x[kp];
        x[kp] = t;
      }
      k -= 2;
    }
  }
}

// M (n x n, n = nu + nc, lower triangle, column-major) = [[R + B^T W, .], [D, -mu I]], the KKT matrix of a stage knot,
// from the staged B (nx x nu) and W = V' B, and the record's R (nu x nu) and D (nc x nu).  No synchronisation.
template <class Ctx>
AB2_RS_HD void kkt_lower(const Ctx &ctx, double *M, const double *Bm, const double *W, const double *R, const double *D,
                         int nx, int nu, int nc, double mu) {
  const int n = nu + nc;
  for (int e = ctx.lane; e < n * n; e += ctx.nl) {
    const int i = e % n, j = e / n;
    if (i < j)
      continue;
    double v;
    if (i < nu) {
      double s = 0.0;
      for (int k = 0; k < nx; ++k)
        s += Bm[k + i * nx] * W[k + j * nx];
      v = R[i + j * nu] + s;
    } else if (j < nu) {
      v = D[(i - nu) + j * nc];
    } else {
      v = i == j ? -mu : 0.0;
    }
    M[e] = v;
  }
}

// Factors the n x n matrix M (lower triangle) in place and solves `cols` columns X + j ld in place, negated with neg
// (each column by one lane).  No synchronisation after the solves.
template <class Ctx>
AB2_RS_HD void kkt_solve(const Ctx &ctx, double *M, double *piv, int n, double *X, int ld, int cols, bool neg) {
  bk_factor(ctx, M, piv, n);
  for (int j = ctx.lane; j < cols; j += ctx.nl) {
    bk_solve(M, piv, n, X + j * ld);
    if (neg)
      for (int i = 0; i < n; ++i)
        X[j * ld + i] = -X[j * ld + i];
  }
}

} // namespace rs

// One work item: instance b, right-hand sides [j0, j0 + R).  sm: resolve_item_doubles(..., a.chunk) doubles.
template <class Ctx>
AB2_RS_HD void resolve_item(const ResolveArgs &a, const Ctx &ctx, double *sm, long b, int j0, int R) {
  const int nx = a.nx, nu = a.nu, nc = a.nc, nct = a.nct, nc0 = a.nc0, N = a.N;
  const int n = nu + nc, n0 = nx + nc0, nr = nu + nc + nx, m = resolve_nkkt(nu, nc, nx, nc0);
  const long B = a.batch;
  const double mu = a.mueq_b ? a.mueq_b[b] : a.mueq;
  const StageOffsets so = stage_offsets(nx, nu, nc);
  double *V = sm, *FB = V + nx * nx, *Bm = FB + nr * nx, *W = Bm + nx * nu, *KKT = W + nx * nu, *piv = KKT + n * n;
  double *K0 = sm, *piv0 = K0 + n0 * n0; // the initial saddle system, over the dead stage buffers
  double *X = sm + resolve_mat_doubles(nx, nu, nc, nc0), *Y = X + a.chunk * nx, *VP = Y + a.chunk * nx, *VX = VP + a.chunk * nx, *S = VX + a.chunk * nx;
  // per right-hand side j of the chunk: X[j] = x, Y[j] = x+, VP[j] = v+, VX[j] = vx, S[j] = solve vector (m)
  auto rix = [&](int j, long per) -> long { return ((long)(j0 + j) * B + b) * per; }; // start of rhs j's block

  // ---- terminal knot: z_N = d_N / mu, vx_N = q_N + C_N^T z_N ----
  {
    const double *CN = a.term + b * a.trec + term_offsets(nx, nct).C;
    for (int e = ctx.lane; e < R * nct; e += ctx.nl) {
      const int j = e / nct, i = e % nct;
      a.vsT[rix(j, nct) + i] = (a.dN ? a.dN[rix(j, nct) + i] : 0.0) / mu;
    }
    for (int e = ctx.lane; e < R * nx; e += ctx.nl) {
      const int j = e / nx, i = e % nx;
      double s = a.q ? a.q[rix(j, (long)(N + 1) * nx) + (long)N * nx + i] : 0.0;
      for (int c = 0; c < nct; ++c)
        s += CN[c + i * nct] * ((a.dN ? a.dN[rix(j, nct) + c] : 0.0) / mu);
      VX[j * nx + i] = s;
    }
    ctx.sync();
  }

  // ---- stage knots, backward ----
  for (int t = N - 1; t >= 0; --t) {
    const double *rec = a.stage + ((long)b * N + ring_slot(t, a.stage_head, N)) * a.srec;
    const double *Br = rec + so.B, *Sr = rec + so.S, *Cr = rec + so.C;
    // the backward pass needs A, S and C instead of the gains: they take the FB rows' place (the same nr * nx doubles)
    double *Am = FB, *Sm = Am + nx * nx, *Cm = Sm + nx * nu;
    rs::load_v(a, ctx, b, t + 1, V);
    for (int e = ctx.lane; e < nx * nx; e += ctx.nl)
      Am[e] = rec[e];
    for (int e = ctx.lane; e < nx * nu; e += ctx.nl)
      Sm[e] = Sr[e];
    for (int e = ctx.lane; e < nc * nx; e += ctx.nl)
      Cm[e] = Cr[e];
    for (int e = ctx.lane; e < nx * nu; e += ctx.nl)
      Bm[e] = Br[e];
    for (int e = ctx.lane; e < R * nx; e += ctx.nl) { // vx_{t+1} is parked in lams[t]
      const int j = e / nx, i = e % nx;
      a.lams[rix(j, (long)N * nx) + (long)t * nx + i] = VX[j * nx + i];
    }
    ctx.sync();
    // W = V' B; v+ = vx_{t+1} + V' f_t
    for (int e = ctx.lane; e < nx * nu; e += ctx.nl) {
      const int i = e % nx, c = e / nx;
      double s = 0.0;
      for (int k = 0; k < nx; ++k)
        s += V[i + k * nx] * Bm[k + c * nx];
      W[e] = s;
    }
    for (int e = ctx.lane; e < R * nx; e += ctx.nl) {
      const int j = e / nx, i = e % nx;
      const double *f = a.f ? a.f + rix(j, (long)N * nx) + (long)t * nx : nullptr;
      double s = 0.0;
      if (f)
        for (int k = 0; k < nx; ++k)
          s += V[i + k * nx] * f[k];
      VP[j * nx + i] = VX[j * nx + i] + s;
    }
    ctx.sync();
    // KKT (lower) = [[R + B^T V' B, .], [D, -mu I]]; solve vector [r_t + B^T v+; d_t]
    rs::kkt_lower(ctx, KKT, Bm, W, rec + so.R, rec + so.D, nx, nu, nc, mu);
    for (int e = ctx.lane; e < R * n; e += ctx.nl) {
      const int j = e / n, i = e % n;
      double v;
      if (i < nu) {
        double s = a.r ? a.r[rix(j, (long)N * nu) + (long)t * nu + i] : 0.0;
        for (int k = 0; k < nx; ++k)
          s += Bm[k + i * nx] * VP[j * nx + k];
        v = s;
      } else {
        v = a.d ? a.d[rix(j, (long)N * nc) + (long)t * nc + (i - nu)] : 0.0;
      }
      S[j * m + i] = v;
    }
    ctx.sync();
    rs::kkt_solve(ctx, KKT, piv, n, S, m, R, true);
    ctx.sync();
    // k -> us[t], z -> vs[t]; a = f + B k -> xs[t+1]; Y = V' B k
    for (int e = ctx.lane; e < R * n; e += ctx.nl) {
      const int j = e / n, i = e % n;
      if (i < nu)
        a.us[rix(j, (long)N * nu) + (long)t * nu + i] = S[j * m + i];
      else
        a.vs[rix(j, (long)N * nc) + (long)t * nc + (i - nu)] = S[j * m + i];
    }
    for (int e = ctx.lane; e < R * nx; e += ctx.nl) {
      const int j = e / nx, i = e % nx;
      double s = a.f ? a.f[rix(j, (long)N * nx) + (long)t * nx + i] : 0.0;
      for (int c = 0; c < nu; ++c)
        s += Bm[i + c * nx] * S[j * m + c];
      a.xs[rix(j, (long)(N + 1) * nx) + (long)(t + 1) * nx + i] = s;
      double w = 0.0;
      for (int c = 0; c < nu; ++c)
        w += W[i + c * nx] * S[j * m + c];
      Y[j * nx + i] = w;
    }
    ctx.sync();
    // vx_t = (qhat + Shat k) + C^T z with qhat = q + A^T v+ and Shat k = S k + A^T V' B k, in the reference's order
    for (int e = ctx.lane; e < R * nx; e += ctx.nl) {
      const int j = e / nx, i = e % nx;
      const double *Ai = Am + i * nx, *kz = S + j * m;
      double qh = 0.0;
      for (int k = 0; k < nx; ++k)
        qh += Ai[k] * VP[j * nx + k];
      qh += a.q ? a.q[rix(j, (long)(N + 1) * nx) + (long)t * nx + i] : 0.0;
      double sk = 0.0;
      for (int k = 0; k < nx; ++k)
        sk += Ai[k] * Y[j * nx + k];
      for (int c = 0; c < nu; ++c)
        sk += Sm[i + c * nx] * kz[c];
      double cz = 0.0;
      for (int c = 0; c < nc; ++c)
        cz += Cm[c + i * nc] * kz[nu + c];
      VX[j * nx + i] = (qh + sk) + cz;
    }
    ctx.sync();
  }

  // ---- initial saddle system [[Vxx_0, G0^T], [G0, 0]] [x_0; lam_0] = -[vx_0; g0] ----
  {
    const double *G0 = a.G0 ? a.G0 + b * nc0 * nx : nullptr;
    for (int e = ctx.lane; e < n0 * n0; e += ctx.nl) {
      const int i = e % n0, j = e / n0;
      if (i < j)
        continue;
      K0[i + j * n0] = i < nx ? rs::vxx_lower(a, b, 0, i, j) : (j < nx ? G0[(i - nx) + j * nc0] : 0.0);
    }
    for (int e = ctx.lane; e < R * n0; e += ctx.nl) {
      const int j = e / n0, i = e % n0;
      S[j * m + i] = i < nx ? -VX[j * nx + i] : -(a.g0 ? a.g0[rix(j, nc0) + (i - nx)] : 0.0);
    }
    ctx.sync();
    rs::kkt_solve(ctx, K0, piv0, n0, S, m, R, false); // the right-hand side is negated already
    ctx.sync();
    for (int e = ctx.lane; e < R * n0; e += ctx.nl) {
      const int j = e / n0, i = e % n0;
      if (i < nx) {
        X[j * nx + i] = S[j * m + i];
        a.xs[rix(j, (long)(N + 1) * nx) + i] = S[j * m + i];
      } else {
        a.lam0[rix(j, nc0) + (i - nx)] = S[j * m + i];
      }
    }
    ctx.sync();
  }

  // ---- forward: u = k + K x, v = z + Z x, x+ = a + Ahat x, lam_{t+1} = vx_{t+1} + Vxx_{t+1} x+ ----
  for (int t = 0; t < N; ++t) {
    const double *fbk = a.fb + (b * N + t) * (long)nr * nx;
    rs::load_v(a, ctx, b, t + 1, V);
    for (int e = ctx.lane; e < nr * nx; e += ctx.nl)
      FB[e] = fbk[e];
    ctx.sync();
    for (int e = ctx.lane; e < R * nr; e += ctx.nl) {
      const int j = e / nr, i = e % nr;
      const double *x = X + j * nx, *row = FB + i * nx;
      double s = 0.0;
      for (int c = 0; c < nx; ++c)
        s += row[c] * x[c];
      if (i < nu) {
        double *o = a.us + rix(j, (long)N * nu) + (long)t * nu + i;
        *o = *o + s;
      } else if (i < nu + nc) {
        double *o = a.vs + rix(j, (long)N * nc) + (long)t * nc + (i - nu);
        *o = *o + s;
      } else {
        double *o = a.xs + rix(j, (long)(N + 1) * nx) + (long)(t + 1) * nx + (i - nu - nc);
        *o = *o + s;
        Y[j * nx + (i - nu - nc)] = *o;
      }
    }
    ctx.sync();
    for (int e = ctx.lane; e < R * nx; e += ctx.nl) {
      const int j = e / nx, i = e % nx;
      double s = 0.0;
      for (int c = 0; c < nx; ++c)
        s += V[i + c * nx] * Y[j * nx + c];
      double *o = a.lams + rix(j, (long)N * nx) + (long)t * nx + i;
      *o = *o + s;
      X[j * nx + i] = Y[j * nx + i];
    }
    ctx.sync();
  }
  // terminal: v_N = z_N + Z_N x_N
  for (int e = ctx.lane; e < R * nct; e += ctx.nl) {
    const int j = e / nct, i = e % nct;
    const double *row = a.fbT + b * nct * nx + (long)i * nx;
    double s = 0.0;
    for (int c = 0; c < nx; ++c)
      s += row[c] * X[j * nx + c];
    double *o = a.vsT + rix(j, nct) + i;
    *o = *o + s;
  }
}

} // namespace ab2
