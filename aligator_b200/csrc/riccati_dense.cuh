// riccati_dense.cuh -- the STAGE-DENSE Riccati solver (gar::DenseKernel, gar/dense-kernel.hpp:55-211;
// gar::RiccatiSolverDense, gar/dense-riccati.hxx:47-123) for a batch, one CTA per instance.
//
// The reference's second algorithm for the same LQ problem: per knot ONE Bunch-Kaufman
// factorisation of the (nu + nc + 2 nx)^2 matrix
//     [[R, D^T, B^T, 0], [D, -mu I, 0, 0], [B, 0, 0, -I], [0, 0, -I, P']]       (dense-kernel.hpp:98-113)
// with right-hand sides -[r; d; f; p'] and -[S^T; C; A; 0]; the solution rows are [k; z; l; y] and
// [K; Z; L; Y] (u = k + K x, v = z + Z x, lbda' = l + L x, x' = y + Y x).  It is not the fast
// path (the proximal kernel's reduced (nu + nc)^2 system is): it exists because the reference
// offers it (LQSolverChoice::STAGEDENSE) and as an independent cross-check on the device.
// Everything in shared memory, thread-per-row Bunch-Kaufman (bk_factor_group over the CTA),
// thread-per-column solves, plain thread-parallel loops for the products.
// Compiles for the host (tests/emu/block_emu.cpp).
#pragma once

#include "riccati_block.cuh"

namespace ab2 {

struct DenseDims {
  int nx, nu, nc, nct, nc0, n; // n = nu + nc + 2 nx
  int srec, trec;
  int s_kkt, s_rhs, s_work, s_aux, s_pn, s_pxn, s_x, s_end; // doubles
};

AB2_HD constexpr DenseDims make_dense_dims(int nx, int nu, int nc, int nct, int nc0) {
  DenseDims d{};
  d.nx = nx;
  d.nu = nu;
  d.nc = nc;
  d.nct = nct;
  d.nc0 = nc0;
  d.n = nu + nc + 2 * nx;
  d.srec = blk_ev(2 * nx * nx + 2 * nx * nu + nu * nu + 2 * nx + nu + nc * (nx + nu + 1));
  d.trec = nx * nx + nx + nct * nx + nct;
  const int n0 = nx + nc0;
  const int nmax = d.n > n0 ? d.n : n0;
  int o = 0;
  d.s_kkt = o;
  o += blk_ev(nmax * nmax);
  d.s_rhs = o; // n x (nx + 1), column-major: column j < nx = feedback column j, column nx = feedforward
  o += blk_ev(nmax * (nx + 1));
  d.s_work = o;
  o += blk_ev(nmax * (nx + 1));
  d.s_aux = o; // dd, sd (nmax each), perm, kind (ints)
  o += 3 * nmax + 2;
  d.s_pn = o; // P' (nx x nx, column-major)
  o += blk_ev(nx * nx);
  d.s_pxn = o;
  o += blk_ev(nx);
  d.s_x = o; // forward: x_t, x_{t+1}
  o += 2 * blk_ev(nx);
  d.s_end = blk_ev(o);
  return d;
}

// mu: where this instance's mu is read (ScalarMu / InstanceMu, riccati_group.cuh).
template <class Ctx, class Mu = ScalarMu>
AB2_D void riccati_dense_sweep(Ctx &ctx, const SweepParams &p, const DenseDims &d, const int inst,
                               double *__restrict__ sm, const Mu &mu = Mu()) {
  const int nx = d.nx, nu = d.nu, nc = d.nc, n = d.n, N = p.N, nct = p.nct, nc0 = p.nc0;
  const int tid = ctx.tid, T = ctx.nthreads;
  const int o2 = nu + nc, o3 = o2 + nx; // row offsets of the l / y blocks
  double *kkt = sm + d.s_kkt, *rhs = sm + d.s_rhs, *work = sm + d.s_work;
  const int nmax = n > nx + nc0 ? n : nx + nc0;
  double *dd = sm + d.s_aux, *sd = dd + nmax;
  int *perm = reinterpret_cast<int *>(sd + nmax), *kind = perm + nmax;
  double *Pn = sm + d.s_pn, *pxn = sm + d.s_pxn;
  const double *stage_b = p.stage + (size_t)inst * N * d.srec;
  double *ff_b = p.ff + (size_t)inst * N * n;
  double *fb_b = p.fb + (size_t)inst * N * n * nx;
  double *Vxx_b = p.Vxx + (size_t)inst * (N + 1) * nx * nx;
  double *vx_b = p.vx + (size_t)inst * (N + 1) * nx;
  CtaAsGroup<Ctx> grp{ctx, tid, T};

  if (p.do_bwd) {
    int st = ST_OK, pv = 0;
    // ---- terminal knot (nu = 0, nx2 = 0): the dense matrix is -mu I (dense-kernel.hpp:55-95)
    {
      const double *tr = p.term + (size_t)inst * d.trec;
      const double *Qt = tr, *qt = tr + nx * nx, *Ct = qt + nx, *dt = Ct + (size_t)nct * nx;
      for (int m = tid; m < nct * nx; m += T) {
        const int r = m / nx, j = m % nx;
        p.fbT[(size_t)inst * nct * nx + m] = Ct[r + (size_t)j * nct] / mu(p, inst);
      }
      for (int m = tid; m < nct; m += T)
        p.ffT[(size_t)inst * nct + m] = dt[m] / mu(p, inst);
      for (int e = tid; e < nx * nx; e += T) { // Pxx = Q + C^T Z
        const int i = e % nx, j = e / nx;
        double acc = 0.0;
        for (int m = 0; m < nct; ++m)
          acc += Ct[m + (size_t)i * nct] * (Ct[m + (size_t)j * nct] / mu(p, inst));
        const double s = Qt[e] + acc;
        Pn[e] = s;
        Vxx_b[(size_t)N * nx * nx + e] = s;
      }
      for (int i = tid; i < nx; i += T) {
        double acc = 0.0;
        for (int m = 0; m < nct; ++m)
          acc += Ct[m + (size_t)i * nct] * (dt[m] / mu(p, inst));
        const double s = qt[i] + acc;
        pxn[i] = s;
        vx_b[(size_t)N * nx + i] = s;
      }
      ctx.sync();
    }
    // ---- stage knots N-1 .. 0 (dense-kernel.hpp:97-175)
    for (int t = N - 1; t >= 0; --t) {
      const double *rec = stage_b + (size_t)t * d.srec;
      const double *A = rec, *Bm = A + nx * nx, *f = Bm + nx * nu, *Q = f + nx, *S = Q + nx * nx, *R = S + nx * nu,
                   *q = R + nu * nu, *r = q + nx, *Cm = r + nu, *Dm = Cm + nc * nx, *dv = Dm + nc * nu;
      for (int e = tid; e < n * n; e += T) { // (:99-113)
        const int i = e % n, j = e / n;
        double v = 0.0;
        const int bi = i < nu ? 0 : (i < o2 ? 1 : (i < o3 ? 2 : 3)), bj = j < nu ? 0 : (j < o2 ? 1 : (j < o3 ? 2 : 3));
        const int ii = i - (bi == 0 ? 0 : (bi == 1 ? nu : (bi == 2 ? o2 : o3)));
        const int jj = j - (bj == 0 ? 0 : (bj == 1 ? nu : (bj == 2 ? o2 : o3)));
        if (bi == 0 && bj == 0)
          v = R[ii + jj * nu];
        else if (bi == 1 && bj == 0)
          v = Dm[ii + jj * nc];
        else if (bi == 0 && bj == 1)
          v = Dm[jj + ii * nc];
        else if (bi == 1 && bj == 1)
          v = (ii == jj) ? -mu(p, inst) : 0.0;
        else if (bi == 2 && bj == 0)
          v = Bm[ii + jj * nx];
        else if (bi == 0 && bj == 2)
          v = Bm[jj + ii * nx];
        else if ((bi == 2 && bj == 3) || (bi == 3 && bj == 2))
          v = (ii == jj) ? -1.0 : 0.0;
        else if (bi == 3 && bj == 3)
          v = Pn[ii + jj * nx];
        kkt[e] = v;
      }
      for (int e = tid; e < n * (nx + 1); e += T) { // right-hand sides (:117-139), column nx = feedforward
        const int i = e % n, j = e / n;
        double v;
        if (j == nx)
          v = i < nu ? -r[i] : (i < o2 ? -dv[i - nu] : (i < o3 ? -f[i - o2] : -pxn[i - o3]));
        else
          v = i < nu ? -S[j + i * nx] : (i < o2 ? -Cm[(i - nu) + j * nc] : (i < o3 ? -A[(i - o2) + j * nx] : 0.0));
        rhs[e] = v;
      }
      ctx.sync();
      if (!bk_factor_group<8>(grp, kkt, n, n, dd, sd, perm, kind, pv))
        st |= ST_STAGE_FACTOR_FAILED;
      for (int j0 = 0; j0 <= nx; j0 += T) {
        const int j = j0 + tid;
        if (j <= nx)
          bk_solve_column_rt(kkt, n, dd, sd, perm, kind, rhs + (size_t)j * n, work + (size_t)j * n, rhs + (size_t)j * n, 1,
                             false);
      }
      ctx.sync();
      double *fft = ff_b + (size_t)t * n, *fbt = fb_b + (size_t)t * n * nx;
      for (int e = tid; e < n * nx; e += T) // fb row-major [K; Z; L; Y]
        fbt[e] = rhs[(e / nx) + (size_t)(e % nx) * n];
      for (int i = tid; i < n; i += T)
        fft[i] = rhs[i + (size_t)nx * n];
      // value function (:151-153, :167-169): Pxx = Q + S K + C^T Z + A^T L, px = q + S k + C^T z + A^T l
      for (int e = tid; e < nx * (nx + 1); e += T) {
        const int i = e % nx, j = e / nx; // column j (nx = the vector)
        const double *col = rhs + (size_t)j * n;
        double s = (j < nx) ? Q[i + j * nx] : q[i];
        double a = 0.0;
        for (int c = 0; c < nu; ++c)
          a += S[i + c * nx] * col[c];
        s += a;
        a = 0.0;
        for (int c = 0; c < nc; ++c)
          a += Cm[c + i * nc] * col[nu + c];
        s += a;
        a = 0.0;
        for (int c = 0; c < nx; ++c)
          a += A[c + i * nx] * col[o2 + c];
        s += a;
        work[e] = s;
      }
      ctx.sync();
      for (int e = tid; e < nx * nx; e += T) {
        Pn[e] = work[e];
        Vxx_b[(size_t)t * nx * nx + e] = work[e];
      }
      for (int i = tid; i < nx; i += T) {
        pxn[i] = work[nx * nx + i];
        vx_b[(size_t)t * nx + i] = work[nx * nx + i];
      }
      ctx.sync();
    }
    // ---- initial stage (dense-riccati.hxx:66-90): [[Pxx_0, G0^T],[G0, 0]] [x0; lbda0] = -[px_0; g0]
    {
      const int n0 = nx + nc0;
      const double *G0 = p.G0 + (size_t)inst * nc0 * nx, *g0 = p.g0 + (size_t)inst * nc0;
      for (int e = tid; e < n0 * n0; e += T) {
        const int i = e % n0, j = e / n0;
        double v = 0.0;
        if (i < nx && j < nx)
          v = Pn[i + j * nx];
        else if (i >= nx && j < nx)
          v = G0[(i - nx) + (size_t)j * nc0];
        else if (i < nx && j >= nx)
          v = G0[(j - nx) + (size_t)i * nc0];
        kkt[e] = v;
      }
      for (int i = tid; i < n0; i += T)
        rhs[i] = (i < nx) ? -pxn[i] : -g0[i - nx];
      ctx.sync();
      if (!bk_factor_group<8>(grp, kkt, n0, n0, dd, sd, perm, kind, pv))
        st |= ST_INIT_FACTOR_FAILED;
      if (tid == 0)
        bk_solve_column_rt(kkt, n0, dd, sd, perm, kind, rhs, work, rhs, 1, false);
      ctx.sync();
      for (int i = tid; i < n0; i += T)
        p.kkt0[(size_t)inst * n0 + i] = rhs[i];
      ctx.sync();
    }
    if (tid == 0) {
      p.status[inst] = st;
      if (p.pivstat)
        p.pivstat[inst] = pv;
    }
  }

  // ---- forward (dense-riccati.hxx:101-123, dense-kernel.hpp:177-215)
  if (p.do_fwd) {
    const int n0 = nx + nc0;
    const double *k0 = p.kkt0 + (size_t)inst * n0;
    double *xs_b = p.xs + (size_t)inst * (N + 1) * nx, *us_b = p.us + (size_t)inst * N * nu,
           *vs_b = p.vs + (size_t)inst * N * nc, *lb_b = p.lbdas + (size_t)inst * N * nx;
    double *xc = sm + d.s_x, *xn = xc + blk_ev(nx);
    ctx.sync();
    for (int i = tid; i < nx; i += T) {
      xc[i] = k0[i];
      xs_b[i] = k0[i];
    }
    for (int m = tid; m < nc0; m += T)
      p.lbd0[(size_t)inst * nc0 + m] = k0[nx + m];
    ctx.sync();
    for (int t = 0; t < N; ++t) {
      const double *fft = ff_b + (size_t)t * n, *fbt = fb_b + (size_t)t * n * nx;
      for (int r = tid; r < n; r += T) {
        double a = 0.0;
        for (int c = 0; c < nx; ++c)
          a += fbt[(size_t)r * nx + c] * xc[c];
        const double v = fft[r] + a;
        if (r < nu)
          us_b[(size_t)t * nu + r] = v;
        else if (r < o2)
          vs_b[(size_t)t * nc + (r - nu)] = v;
        else if (r < o3)
          lb_b[(size_t)t * nx + (r - o2)] = v; // lbda_{t+1}
        else {
          xn[r - o3] = v;
          xs_b[(size_t)(t + 1) * nx + (r - o3)] = v;
        }
      }
      ctx.sync();
      double *tmp = xc;
      xc = xn;
      xn = tmp;
    }
    for (int m = tid; m < nct; m += T) { // terminal multipliers v_N = z + Z x_N
      double s = p.ffT[(size_t)inst * nct + m];
      for (int c = 0; c < nx; ++c)
        s += p.fbT[(size_t)inst * nct * nx + (size_t)m * nx + c] * xc[c];
      p.vsT[(size_t)inst * nct + m] = s;
    }
    ctx.sync();
  }
}

} // namespace ab2
