// lq_factor_adjoint.cuh -- reverse mode of the backward recursion (ab2_gar_factor_adjoint, include/aligator_b200/gar.h):
// gradients of the problem records for cotangents of the factorisation FF, FB, VXX, VX, FFT, FBT.  Plain C++ apart
// from the execution context, so that the host emulation (tests/emu/factor_adjoint_emu.cpp) compiles the same program.
//
// Vxx_t and vx_t are read only by knot t-1, so the reverse pass runs FORWARD in time: one work item (instance b)
// carries Vbar, vbar (the cotangents of Vxx_t, vx_t; Vbar symmetric) from knot 0 to the terminal knot.  Per stage knot
// the forward quantities are recomputed from the record and the stored factor: V' = Vxx_{t+1}, v' = vx_{t+1},
// X = [[K, k], [Z, z]], Shat = S + A^T V' B, v+ = v' + V' f, and M = [[R + B^T V' B, D^T], [D, -mu I]], factored again
// by Bunch-Kaufman from its lower triangle as resolve does.  With sym(M) = (M + M^T) / 2 and cotangents of the
// knot's outputs marked 0:
//   closed loop  Kb = Kb0 + B^T Ahatb,  kb = kb0 + B^T ab,  Bb = Ahatb K^T + ab k^T,  Ab = Ahatb,  fb = ab
//   value        Qb = Vbar,  qb = vbar,  Shatb = Vbar K^T + vbar k^T,  Kb += Shat^T Vbar,  kb += Shat^T vbar
//                Cb = Z Vbar + z vbar^T,  Zb = Zb0 + C Vbar,  zb = zb0 + C vbar
//   solve        P = -M^-1 [[Kb, kb], [Zb, zb]]  (P_u: the first nu rows, P_c: the last nc rows)
//                Shatb += P_u[:, :nx]^T,  rb = P_u[:, nx],  Cb += P_c[:, :nx],  db = P_c[:, nx]
//                Rb = sym(P_u X_u^T),  Db = P_c X_u^T + X_c P_u^T  (X_u = [K, k], X_c = [Z, z]),  Sb = Shatb
//   products     Ab += 2 V' A Qb + V' B Shatb^T + v+ qb^T,  Bb += 2 V' B Rb + V' A Shatb + v+ rb^T
//                vb+ = A qb + B rb,  fb += V' vb+
//   carry        Vbar <- sym(Vxxb0_{t+1}) + sym(A (Qb A^T + Shatb B^T) + B (Rb B^T) + vb+ f^T),  vbar <- vxb0_{t+1} + vb+
// and at the terminal knot (Z_N = C_N / mu, z_N = d_N / mu as stored in FBT, FFT):
//   Zb = Zb0_N + C_N Vbar,  zb = zb0_N + C_N vbar,  C_Nb = Z_N Vbar + z_N vbar^T + Zb / mu,  d_Nb = zb / mu,
//   Q_Nb = Vbar,  q_Nb = vbar.
// G0 and g0 do not enter the factorisation: their gradient is zero.
//
// Work split: one item per instance, run by `nl` lanes that synchronise with ctx.sync() (one warp, or a whole CTA for
// items too large to share an SM).  Every entry of a result is summed by one lane in a fixed order, and the
// factorisation is resolve's, so the results do not depend on the lane count.
#pragma once

#include "lq_resolve.cuh"

namespace ab2 {

struct FactorAdjointArgs {
  ResolveArgs fac;                  // records and factorisation: dims, stage .. G0, fb, fbT, Vxx, Vxx0, mueq, mueq_b
  const double *ff, *vx, *ffT;      // FF [batch][N][nu+nc+nx], VX [batch][N+1][nx], FFT [batch][nct]
  // cotangents in ab2_gar_get's layouts (vxx full column-major [batch][N+1][nx*nx]); null = zero
  const double *c_ff, *c_fb, *c_vxx, *c_vx, *c_fft, *c_fbt;
  double *g_stage, *g_term, *g_G0, *g_g0; // the problem's layouts; null = not written
};

// doubles of shared memory one item uses: Vbar, V', A, V'A (then Qb A^T + Shatb B^T), Ahatb (then the carry's sum);
// B, V'B (then Rb B^T), Shat (then Shatb); C; [K; Z]; P; M and pivots; Rb; [k; z], vbar, f, v+, ab, vb+
AB2_RS_HD int factor_adjoint_item_doubles(int nx, int nu, int nc) {
  const int n = nu + nc;
  const int d = 5 * nx * nx + 3 * nx * nu + nc * nx + n * nx + n * (nx + 1) + n * n + n + nu * nu + n + 5 * nx;
  return (d + 1) & ~1;
}

template <class Ctx>
AB2_RS_HD void factor_adjoint_item(const FactorAdjointArgs &a, const Ctx &ctx, double *sm, long b) {
  const ResolveArgs &r = a.fac;
  const int nx = r.nx, nu = r.nu, nc = r.nc, nct = r.nct, N = r.N;
  const int n = nu + nc, nr = n + nx, m = nx + 1;
  const double mu = r.mueq_b ? r.mueq_b[b] : r.mueq;
  double *Vb = sm, *Vp = Vb + nx * nx, *Am = Vp + nx * nx, *T = Am + nx * nx, *Ahb = T + nx * nx;
  double *Bm = Ahb + nx * nx, *W = Bm + nx * nu, *Sh = W + nx * nu, *Cm = Sh + nx * nu, *KZ = Cm + nc * nx;
  double *P = KZ + n * nx, *M = P + n * m, *piv = M + n * n, *Rb = piv + n, *kz = Rb + nu * nu;
  double *vb = kz + n, *f = vb + nx, *vp = f + nx, *ab = vp + nx, *vbp = ab + nx;
  // all matrices column-major: Vb, Vp, Am, T, Ahb nx x nx; Bm, W, Sh nx x nu; Cm nc x nx; KZ = [K; Z] n x nx;
  // P n x (nx + 1); M n x n; Rb nu x nu

  // ---- seed: Vbar = sym(Vxxb0_0), vbar = vxb0_0 ----
  {
    const double *cV = a.c_vxx ? a.c_vxx + b * (N + 1) * nx * nx : nullptr;
    for (int e = ctx.lane; e < nx * nx; e += ctx.nl) {
      const int i = e % nx, j = e / nx;
      Vb[e] = cV ? 0.5 * (cV[i + j * nx] + cV[j + i * nx]) : 0.0;
    }
    for (int i = ctx.lane; i < nx; i += ctx.nl)
      vb[i] = a.c_vx ? a.c_vx[b * (N + 1) * nx + i] : 0.0;
    if (a.g_G0)
      for (int e = ctx.lane; e < r.nc0 * nx; e += ctx.nl)
        a.g_G0[b * r.nc0 * nx + e] = 0.0;
    if (a.g_g0)
      for (int e = ctx.lane; e < r.nc0; e += ctx.nl)
        a.g_g0[b * r.nc0 + e] = 0.0;
    ctx.sync();
  }

  for (int t = 0; t < N; ++t) {
    const StageOffsets so = stage_offsets(nx, nu, nc);
    const double *rec = r.stage + ((long)b * N + ring_slot(t, r.stage_head, N)) * r.srec;
    double *g = a.g_stage ? a.g_stage + ((long)b * N + t) * r.srec : nullptr;
    const double *fbk = r.fb + (b * N + t) * (long)nr * nx, *ffk = a.ff + (b * N + t) * (long)nr;
    const double *cfb = a.c_fb ? a.c_fb + (b * N + t) * (long)nr * nx : nullptr;
    const double *cff = a.c_ff ? a.c_ff + (b * N + t) * (long)nr : nullptr;

    // 1. stage the record blocks, V', [K; Z], [k; z], Ahatb, ab, and P = [[Kb0, kb0], [Zb0, zb0]]
    rs::load_v(r, ctx, b, t + 1, Vp);
    for (int e = ctx.lane; e < nx * nx; e += ctx.nl) {
      const int i = e % nx, j = e / nx;
      Am[e] = rec[e];
      Ahb[e] = cfb ? cfb[(n + i) * nx + j] : 0.0;
    }
    for (int e = ctx.lane; e < nx * nu; e += ctx.nl)
      Bm[e] = rec[so.B + e];
    for (int e = ctx.lane; e < nc * nx; e += ctx.nl)
      Cm[e] = rec[so.C + e];
    for (int e = ctx.lane; e < n * m; e += ctx.nl) {
      const int i = e % n, j = e / n;
      if (j < nx) {
        KZ[e] = fbk[i * nx + j];
        P[e] = cfb ? cfb[i * nx + j] : 0.0;
      } else {
        kz[i] = ffk[i];
        P[e] = cff ? cff[i] : 0.0;
      }
    }
    for (int i = ctx.lane; i < nx; i += ctx.nl) {
      f[i] = rec[so.f + i];
      ab[i] = cff ? cff[n + i] : 0.0;
    }
    ctx.sync();
    // 2. W = V' B, T = V' A, v+ = vx_{t+1} + V' f
    for (int e = ctx.lane; e < nx * (nu + nx); e += ctx.nl) {
      const int i = e % nx, c = e / nx;
      const double *X = c < nu ? Bm + c * nx : Am + (c - nu) * nx;
      double s = 0.0;
      for (int k = 0; k < nx; ++k)
        s += Vp[i + k * nx] * X[k];
      (c < nu ? W + c * nx : T + (c - nu) * nx)[i] = s;
    }
    for (int i = ctx.lane; i < nx; i += ctx.nl) {
      double s = 0.0;
      for (int k = 0; k < nx; ++k)
        s += Vp[i + k * nx] * f[k];
      vp[i] = a.vx[(b * (N + 1) + t + 1) * nx + i] + s;
    }
    ctx.sync();
    // 3. Shat = S + A^T W; M (lower) = [[R + B^T W, .], [D, -mu I]]
    for (int e = ctx.lane; e < nx * nu; e += ctx.nl) {
      const int i = e % nx, c = e / nx;
      double s = rec[so.S + e];
      for (int k = 0; k < nx; ++k)
        s += Am[k + i * nx] * W[k + c * nx];
      Sh[e] = s;
    }
    rs::kkt_lower(ctx, M, Bm, W, rec + so.R, rec + so.D, nx, nu, nc, mu);
    ctx.sync();
    // 4. P += [[B^T Ahatb + Shat^T Vbar, B^T ab + Shat^T vbar], [C Vbar, C vbar]]; factor M; P <- -M^-1 P
    for (int e = ctx.lane; e < n * m; e += ctx.nl) {
      const int i = e % n, j = e / n;
      const double *Vj = j < nx ? Vb + j * nx : vb, *Aj = j < nx ? Ahb + j * nx : ab;
      double s = 0.0;
      if (i < nu) {
        for (int k = 0; k < nx; ++k)
          s += Bm[k + i * nx] * Aj[k];
        for (int k = 0; k < nx; ++k)
          s += Sh[k + i * nx] * Vj[k];
      } else {
        for (int k = 0; k < nx; ++k)
          s += Cm[(i - nu) + k * nc] * Vj[k];
      }
      P[e] += s;
    }
    ctx.sync();
    rs::kkt_solve(ctx, M, piv, n, P, n, m, true);
    ctx.sync();
    // 5. Shatb (over Shat), Rb; the gradients of Q, q, r, d, C, D, S
    for (int e = ctx.lane; e < nx * nu; e += ctx.nl) {
      const int i = e % nx, c = e / nx;
      double s = 0.0;
      for (int k = 0; k < nx; ++k)
        s += Vb[i + k * nx] * KZ[c + k * n];
      Sh[e] = (s + vb[i] * kz[c]) + P[c + i * n];
    }
    for (int e = ctx.lane; e < nu * nu; e += ctx.nl) {
      const int i = e % nu, j = e / nu;
      double s1 = 0.0, s2 = 0.0;
      for (int l = 0; l < nx; ++l) {
        s1 += P[i + l * n] * KZ[j + l * n];
        s2 += P[j + l * n] * KZ[i + l * n];
      }
      s1 += P[i + nx * n] * kz[j];
      s2 += P[j + nx * n] * kz[i];
      Rb[e] = 0.5 * (s1 + s2);
    }
    if (g) {
      for (int e = ctx.lane; e < nx * nx; e += ctx.nl)
        g[so.Q + e] = Vb[e];
      for (int i = ctx.lane; i < nx; i += ctx.nl)
        g[so.q + i] = vb[i];
      for (int i = ctx.lane; i < n; i += ctx.nl)
        g[(i < nu ? so.r : so.d - nu) + i] = P[i + nx * n];
      for (int e = ctx.lane; e < nc * nx; e += ctx.nl) { // Cb = Z Vbar + z vbar^T + P_c[:, :nx]
        const int c = e % nc, i = e / nc;
        double s = 0.0;
        for (int k = 0; k < nx; ++k)
          s += KZ[(nu + c) + k * n] * Vb[k + i * nx];
        g[so.C + e] = (s + kz[nu + c] * vb[i]) + P[(nu + c) + i * n];
      }
      for (int e = ctx.lane; e < nc * nu; e += ctx.nl) { // Db = P_c X_u^T + X_c P_u^T
        const int c = e % nc, j = e / nc;
        double s1 = 0.0, s2 = 0.0;
        for (int l = 0; l < m; ++l) {
          const double xu = l < nx ? KZ[j + l * n] : kz[j], xc = l < nx ? KZ[(nu + c) + l * n] : kz[nu + c];
          s1 += P[(nu + c) + l * n] * xu;
          s2 += xc * P[j + l * n];
        }
        g[so.D + e] = s1 + s2;
      }
      if (ctx.lane == 0 && r.srec > so.end)
        g[so.end] = 0.0;
    }
    ctx.sync();
    // 6. Ab, Bb, the gradients of S and R; vb+ = A qb + B rb
    for (int e = ctx.lane; e < nx * nx; e += ctx.nl) {
      const int i = e % nx, j = e / nx;
      double s = 0.0;
      for (int k = 0; k < nx; ++k)
        s += T[i + k * nx] * Vb[k + j * nx];
      double w = 0.0;
      for (int c = 0; c < nu; ++c)
        w += W[i + c * nx] * Sh[j + c * nx];
      if (g)
        g[e] = ((Ahb[e] + 2.0 * s) + w) + vp[i] * vb[j];
    }
    for (int e = ctx.lane; e < nx * nu; e += ctx.nl) {
      const int i = e % nx, c = e / nx;
      double s = 0.0;
      for (int k = 0; k < nx; ++k)
        s += Ahb[i + k * nx] * KZ[c + k * n];
      double w = 0.0;
      for (int j = 0; j < nu; ++j)
        w += W[i + j * nx] * Rb[j + c * nu];
      double h = 0.0;
      for (int k = 0; k < nx; ++k)
        h += T[i + k * nx] * Sh[k + c * nx];
      if (g) {
        g[so.B + e] = (((s + ab[i] * kz[c]) + 2.0 * w) + h) + vp[i] * P[c + nx * n];
        g[so.S + e] = Sh[e];
      }
    }
    if (g)
      for (int e = ctx.lane; e < nu * nu; e += ctx.nl)
        g[so.R + e] = Rb[e];
    for (int i = ctx.lane; i < nx; i += ctx.nl) {
      double s = 0.0;
      for (int k = 0; k < nx; ++k)
        s += Am[i + k * nx] * vb[k];
      for (int c = 0; c < nu; ++c)
        s += Bm[i + c * nx] * P[c + nx * n];
      vbp[i] = s;
    }
    ctx.sync();
    // 7. fb = ab + V' vb+; T <- Qb A^T + Shatb B^T; W <- (Rb B^T)^T = B Rb (nx x nu)
    if (g)
      for (int i = ctx.lane; i < nx; i += ctx.nl) {
        double s = 0.0;
        for (int k = 0; k < nx; ++k)
          s += Vp[i + k * nx] * vbp[k];
        g[so.f + i] = ab[i] + s;
      }
    for (int e = ctx.lane; e < nx * nx; e += ctx.nl) {
      const int i = e % nx, j = e / nx;
      double s = 0.0;
      for (int k = 0; k < nx; ++k)
        s += Vb[i + k * nx] * Am[j + k * nx];
      for (int c = 0; c < nu; ++c)
        s += Sh[i + c * nx] * Bm[j + c * nx];
      T[e] = s;
    }
    for (int e = ctx.lane; e < nx * nu; e += ctx.nl) {
      const int i = e % nx, c = e / nx;
      double s = 0.0;
      for (int j = 0; j < nu; ++j)
        s += Bm[i + j * nx] * Rb[j + c * nu];
      W[e] = s;
    }
    ctx.sync();
    // 8. Ahb <- A T + (B Rb) B^T + vb+ f^T
    for (int e = ctx.lane; e < nx * nx; e += ctx.nl) {
      const int i = e % nx, j = e / nx;
      double s = 0.0;
      for (int k = 0; k < nx; ++k)
        s += Am[i + k * nx] * T[k + j * nx];
      double w = 0.0;
      for (int c = 0; c < nu; ++c)
        w += W[i + c * nx] * Bm[j + c * nx];
      Ahb[e] = (s + w) + vbp[i] * f[j];
    }
    ctx.sync();
    // 9. carry: Vbar <- sym(Vxxb0_{t+1}) + sym(Ahb), vbar <- vxb0_{t+1} + vb+
    {
      const double *cV = a.c_vxx ? a.c_vxx + (b * (N + 1) + t + 1) * nx * nx : nullptr;
      for (int e = ctx.lane; e < nx * nx; e += ctx.nl) {
        const int i = e % nx, j = e / nx;
        const double s = 0.5 * (Ahb[i + j * nx] + Ahb[j + i * nx]);
        Vb[e] = cV ? 0.5 * (cV[i + j * nx] + cV[j + i * nx]) + s : s;
      }
      for (int i = ctx.lane; i < nx; i += ctx.nl)
        vb[i] = a.c_vx ? a.c_vx[(b * (N + 1) + t + 1) * nx + i] + vbp[i] : vbp[i];
    }
    ctx.sync();
  }

  // ---- terminal knot ----
  if (a.g_term) {
    const TermOffsets to = term_offsets(nx, nct);
    const double *rec = r.term + b * r.trec, *CN = rec + to.C;
    const double *ZN = r.fbT + b * nct * nx, *zN = a.ffT + b * nct;
    double *g = a.g_term + b * r.trec;
    for (int e = ctx.lane; e < nx * nx; e += ctx.nl)
      g[e] = Vb[e];
    for (int i = ctx.lane; i < nx; i += ctx.nl)
      g[to.q + i] = vb[i];
    for (int e = ctx.lane; e < nct * nx; e += ctx.nl) { // C_Nb = Z_N Vbar + z_N vbar^T + Zb / mu
      const int c = e % nct, i = e / nct;
      double s = 0.0, z = a.c_fbt ? a.c_fbt[b * nct * nx + c * nx + i] : 0.0;
      for (int k = 0; k < nx; ++k)
        s += ZN[c * nx + k] * Vb[k + i * nx];
      for (int k = 0; k < nx; ++k)
        z += CN[c + k * nct] * Vb[k + i * nx];
      g[to.C + e] = (s + zN[c] * vb[i]) + z / mu;
    }
    for (int c = ctx.lane; c < nct; c += ctx.nl) { // d_Nb = (zb0_N + C_N vbar) / mu
      double z = a.c_fft ? a.c_fft[b * nct + c] : 0.0;
      for (int k = 0; k < nx; ++k)
        z += CN[c + k * nct] * vb[k];
      g[to.d + c] = z / mu;
    }
  }
}

} // namespace ab2
