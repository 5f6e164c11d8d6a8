// lq_theta.cuh -- derivatives of a parametric LQ solution with respect to theta (ab2_gar_theta_tangent and
// ab2_gar_theta_adjoint, include/aligator_b200/gar.h).  Plain C++ apart from the execution context, so that the host
// emulation (tests/emu/theta_emu.cpp) compiles the same programs and runs them on emulated lanes.
//
// The matrices of a parametric problem do not depend on theta, so its solution is affine in theta, z(theta) = z_0 +
// J theta, and J is made of factors the last backward left in HBM: the gains FB = [K; Z; Ahat], the theta gains
// FTH = [Kth; Zth; Yth], the cost-to-go Hessians Vxx and their theta columns Vxt, the terminal gain Z_N (FBT) and the
// initial system's theta columns F0 = KKT0FTH (rows x_0, then lam_0).
//   tangent (forward in time), direction d in R^nth -- the theta terms of the parametric forward pass:
//     x^_0 = F0_x d,  lam^_0 = F0_lam d
//     t = 0..N-1:  u^_t = K_t x^_t + Kth_t d,  v^_t = Z_t x^_t + Zth_t d,  x^_{t+1} = Ahat_t x^_t + Yth_t d,
//                  lam^_{t+1} = Vxx_{t+1} x^_{t+1} + Vxt_{t+1} d
//     v^_N = Z_N x^_N   (the terminal knot has no theta term)
//   adjoint (its exact transpose, backward in time), cotangents (xbar, ubar, vbar, vbar_N, lambar_0, lambar), with c_t
//   the cotangent of x_t:
//     c_N = xbar_N + Z_N^T vbar_N + Vxx_N lambar_N,   thbar = Vxt_N^T lambar_N           (the Vxx, Vxt terms: N >= 1)
//     t = N-1..0:  thbar += Kth_t^T ubar_t + Zth_t^T vbar_t + Yth_t^T c_{t+1} (+ Vxt_t^T lambar_t, t >= 1)
//                  c_t = xbar_t + K_t^T ubar_t + Z_t^T vbar_t + Ahat_t^T c_{t+1} (+ Vxx_t lambar_t, t >= 1)
//     thbar += F0_x^T c_0 + F0_lam^T lambar_0
// Both read the stored matrices as they are (Vxx_t in the full [batch][N+1][nx*nx] blocks of the CTA-per-instance
// kernel, which every parametric handle runs), and the adjoint applies the transpose of each, so the two are each
// other's transpose to rounding.
//
// Work split: one item per (instance, chunk of directions), run by `nl` lanes that synchronise with ctx.sync() (one
// warp on the device).  A knot's FB, FTH, Vxx and Vxt are staged once per item and shared by the chunk; each entry of
// a result is computed by one lane in a fixed order and nothing is accumulated across lanes, so a direction's result
// does not depend on the chunk it shares, its position in it, or the lane count.
#pragma once

#if defined(__CUDACC__)
#define AB2_TH_HD __host__ __device__ __forceinline__
#else
#define AB2_TH_HD inline
#endif

namespace ab2 {

struct ThetaArgs {
  int batch, N, nx, nu, nc, nct, nc0, nth;
  int nrhs, chunk;                        // directions, and how many one item holds on chip
  const double *fb, *fth, *fbT;           // FB [batch][N][nr*nx], FTH [batch][N][nr*nth] (row-major), FBT [batch][nct*nx]
  const double *Vxx, *Vxt;                // [batch][N+1][nx*nx], [batch][N+1][nx*nth] (column-major)
  const double *kkt0fth;                  // [batch][(nx+nc0)*nth] (row-major)
  // tangent: dtheta [nrhs][batch][nth] in, the solution's layouts out ([nrhs][batch][...])
  const double *dtheta;
  double *xs, *us, *vs, *vsT, *lam0, *lams;
  // adjoint: cotangents in the solution's layouts (null = zero), theta_bar [nrhs][batch][nth] out
  const double *cxs, *cus, *cvs, *cvsT, *clam0, *clams;
  double *theta_bar;
};

// doubles of the matrix region: a stage knot's FB, FTH, Vxx, Vxt; the terminal knot's Z_N, Vxx_N, Vxt_N; or F0
AB2_TH_HD int theta_mat_doubles(int nx, int nu, int nc, int nct, int nc0, int nth) {
  const int nr = nu + nc + nx;
  const int stage = nr * nx + nr * nth + nx * nx + nx * nth;
  const int term = nct * nx + nx * nx + nx * nth;
  const int init = (nx + nc0) * nth;
  const int m = stage > term ? stage : term;
  return m > init ? m : init;
}
// doubles of shared memory one item of either program uses: the matrix region, and per direction the adjoint's
// [ubar; vbar; c_{t+1}], lambar_t, c_t and thbar (the tangent uses the first 2 nx + nth of these: x^, x^+, d)
AB2_TH_HD int theta_item_doubles(int nx, int nu, int nc, int nct, int nc0, int nth, int chunk) {
  const int per = (nu + nc + nx) + 2 * nx + nth;
  return ((theta_mat_doubles(nx, nu, nc, nct, nc0, nth) + chunk * per) + 1) & ~1;
}

namespace th {

template <class Ctx> AB2_TH_HD void copy(const Ctx &ctx, double *dst, const double *src, int n) {
  for (int e = ctx.lane; e < n; e += ctx.nl)
    dst[e] = src[e];
}

} // namespace th

// Tangent, one work item: instance b, directions [j0, j0 + R).  sm: theta_item_doubles(..., a.chunk) doubles.
template <class Ctx>
AB2_TH_HD void theta_tangent_item(const ThetaArgs &a, const Ctx &ctx, double *sm, long b, int j0, int R) {
  const int nx = a.nx, nu = a.nu, nc = a.nc, nct = a.nct, nc0 = a.nc0, nth = a.nth, N = a.N;
  const int nk = nu + nc, nr = nk + nx, n0 = nx + nc0;
  const long B = a.batch;
  double *FB = sm, *FT = FB + nr * nx, *V = FT + nr * nth, *VT = V + nx * nx;
  double *X = sm + theta_mat_doubles(nx, nu, nc, nct, nc0, nth), *Y = X + a.chunk * nx, *D = Y + a.chunk * nx;
  // per direction j of the chunk: X[j] = x^_t, Y[j] = x^_{t+1}, D[j] = d
  auto rix = [&](int j, long per) -> long { return ((long)(j0 + j) * B + b) * per; }; // start of direction j's block

  // ---- initial: x^_0 = F0_x d, lam^_0 = F0_lam d ----
  for (int e = ctx.lane; e < R * nth; e += ctx.nl) {
    const int j = e / nth, c = e % nth;
    D[j * nth + c] = a.dtheta[rix(j, nth) + c];
  }
  th::copy(ctx, FB, a.kkt0fth + b * n0 * nth, n0 * nth);
  ctx.sync();
  for (int e = ctx.lane; e < R * n0; e += ctx.nl) {
    const int j = e / n0, i = e % n0;
    double s = 0.0;
    for (int c = 0; c < nth; ++c)
      s += FB[i * nth + c] * D[j * nth + c];
    if (i < nx) {
      X[j * nx + i] = s;
      a.xs[rix(j, (long)(N + 1) * nx) + i] = s;
    } else {
      a.lam0[rix(j, nc0) + (i - nx)] = s;
    }
  }
  ctx.sync();

  // ---- stage knots ----
  for (int t = 0; t < N; ++t) {
    th::copy(ctx, FB, a.fb + (b * N + t) * (long)nr * nx, nr * nx);
    th::copy(ctx, FT, a.fth + (b * N + t) * (long)nr * nth, nr * nth);
    th::copy(ctx, V, a.Vxx + (b * (N + 1) + t + 1) * (long)nx * nx, nx * nx);
    th::copy(ctx, VT, a.Vxt + (b * (N + 1) + t + 1) * (long)nx * nth, nx * nth);
    ctx.sync();
    // [u^; v^; x^+] = FB x^ + FTH d, row r by one lane
    for (int e = ctx.lane; e < R * nr; e += ctx.nl) {
      const int j = e / nr, r = e % nr;
      const double *x = X + j * nx, *d = D + j * nth;
      double s = 0.0;
      for (int c = 0; c < nx; ++c)
        s += FB[r * nx + c] * x[c];
      double acc = 0.0;
      for (int c = 0; c < nth; ++c)
        acc += FT[r * nth + c] * d[c];
      s += acc;
      if (r < nu) {
        a.us[rix(j, (long)N * nu) + (long)t * nu + r] = s;
      } else if (r < nk) {
        a.vs[rix(j, (long)N * nc) + (long)t * nc + (r - nu)] = s;
      } else {
        Y[j * nx + (r - nk)] = s;
        a.xs[rix(j, (long)(N + 1) * nx) + (long)(t + 1) * nx + (r - nk)] = s;
      }
    }
    ctx.sync();
    // lam^_{t+1} = Vxx_{t+1} x^_{t+1} + Vxt_{t+1} d
    for (int e = ctx.lane; e < R * nx; e += ctx.nl) {
      const int j = e / nx, i = e % nx;
      const double *y = Y + j * nx, *d = D + j * nth;
      double s = 0.0;
      for (int c = 0; c < nx; ++c)
        s += V[c * nx + i] * y[c];
      double acc = 0.0;
      for (int c = 0; c < nth; ++c)
        acc += VT[i + c * nx] * d[c];
      a.lams[rix(j, (long)N * nx) + (long)t * nx + i] = s + acc;
    }
    ctx.sync();
    double *tmp = X;
    X = Y;
    Y = tmp;
  }

  // ---- terminal: v^_N = Z_N x^_N ----
  th::copy(ctx, FB, a.fbT + b * nct * nx, nct * nx);
  ctx.sync();
  for (int e = ctx.lane; e < R * nct; e += ctx.nl) {
    const int j = e / nct, m = e % nct;
    double s = 0.0;
    for (int c = 0; c < nx; ++c)
      s += FB[m * nx + c] * X[j * nx + c];
    a.vsT[rix(j, nct) + m] = s;
  }
}

// Adjoint, one work item: instance b, directions [j0, j0 + R).  sm: theta_item_doubles(..., a.chunk) doubles.
template <class Ctx>
AB2_TH_HD void theta_adjoint_item(const ThetaArgs &a, const Ctx &ctx, double *sm, long b, int j0, int R) {
  const int nx = a.nx, nu = a.nu, nc = a.nc, nct = a.nct, nc0 = a.nc0, nth = a.nth, N = a.N;
  const int nk = nu + nc, nr = nk + nx, n0 = nx + nc0;
  const long B = a.batch;
  double *W = sm + theta_mat_doubles(nx, nu, nc, nct, nc0, nth), *L = W + a.chunk * nr, *Cn = L + a.chunk * nx,
         *TB = Cn + a.chunk * nx;
  // per direction j of the chunk: W[j] = [ubar_t; vbar_t; c_{t+1}], L[j] = lambar_t, Cn[j] = c_t, TB[j] = thbar
  auto rix = [&](int j, long per) -> long { return ((long)(j0 + j) * B + b) * per; };
  auto lambar = [&](int j, int t, int i) -> double { // lambar_t (t >= 1) = the cotangent of lams[t - 1]
    return a.clams ? a.clams[rix(j, (long)N * nx) + (long)(t - 1) * nx + i] : 0.0;
  };

  // ---- terminal: c_N = xbar_N + Z_N^T vbar_N + Vxx_N lambar_N, thbar = Vxt_N^T lambar_N ----
  {
    double *ZN = sm, *V = ZN + nct * nx, *VT = V + nx * nx;
    th::copy(ctx, ZN, a.fbT + b * nct * nx, nct * nx);
    if (N >= 1) {
      th::copy(ctx, V, a.Vxx + (b * (N + 1) + N) * (long)nx * nx, nx * nx);
      th::copy(ctx, VT, a.Vxt + (b * (N + 1) + N) * (long)nx * nth, nx * nth);
      for (int e = ctx.lane; e < R * nx; e += ctx.nl)
        L[(e / nx) * nx + e % nx] = lambar(e / nx, N, e % nx);
    }
    ctx.sync();
    for (int e = ctx.lane; e < R * nx; e += ctx.nl) {
      const int j = e / nx, k = e % nx;
      double s = a.cxs ? a.cxs[rix(j, (long)(N + 1) * nx) + (long)N * nx + k] : 0.0;
      if (a.cvsT)
        for (int m = 0; m < nct; ++m)
          s += ZN[m * nx + k] * a.cvsT[rix(j, nct) + m];
      if (N >= 1)
        for (int i = 0; i < nx; ++i)
          s += V[k * nx + i] * L[j * nx + i];
      Cn[j * nx + k] = s;
    }
    for (int e = ctx.lane; e < R * nth; e += ctx.nl) {
      const int j = e / nth, c = e % nth;
      double s = 0.0;
      if (N >= 1)
        for (int i = 0; i < nx; ++i)
          s += VT[i + c * nx] * L[j * nx + i];
      TB[j * nth + c] = s;
    }
    ctx.sync();
  }

  // ---- stage knots, backward ----
  double *FB = sm, *FT = FB + nr * nx, *V = FT + nr * nth, *VT = V + nx * nx;
  for (int t = N - 1; t >= 0; --t) {
    th::copy(ctx, FB, a.fb + (b * N + t) * (long)nr * nx, nr * nx);
    th::copy(ctx, FT, a.fth + (b * N + t) * (long)nr * nth, nr * nth);
    if (t >= 1) {
      th::copy(ctx, V, a.Vxx + (b * (N + 1) + t) * (long)nx * nx, nx * nx);
      th::copy(ctx, VT, a.Vxt + (b * (N + 1) + t) * (long)nx * nth, nx * nth);
      for (int e = ctx.lane; e < R * nx; e += ctx.nl)
        L[(e / nx) * nx + e % nx] = lambar(e / nx, t, e % nx);
    }
    for (int e = ctx.lane; e < R * nr; e += ctx.nl) {
      const int j = e / nr, r = e % nr;
      double w;
      if (r < nu)
        w = a.cus ? a.cus[rix(j, (long)N * nu) + (long)t * nu + r] : 0.0;
      else if (r < nk)
        w = a.cvs ? a.cvs[rix(j, (long)N * nc) + (long)t * nc + (r - nu)] : 0.0;
      else
        w = Cn[j * nx + (r - nk)];
      W[j * nr + r] = w;
    }
    ctx.sync();
    // c_t = xbar_t + FB^T w (+ Vxx_t lambar_t), column k by one lane
    for (int e = ctx.lane; e < R * nx; e += ctx.nl) {
      const int j = e / nx, k = e % nx;
      const double *w = W + j * nr;
      double s = a.cxs ? a.cxs[rix(j, (long)(N + 1) * nx) + (long)t * nx + k] : 0.0;
      for (int r = 0; r < nr; ++r)
        s += FB[r * nx + k] * w[r];
      if (t >= 1)
        for (int i = 0; i < nx; ++i)
          s += V[k * nx + i] * L[j * nx + i];
      Cn[j * nx + k] = s;
    }
    // thbar += FTH^T w (+ Vxt_t^T lambar_t), column c by one lane
    for (int e = ctx.lane; e < R * nth; e += ctx.nl) {
      const int j = e / nth, c = e % nth;
      const double *w = W + j * nr;
      double s = 0.0;
      for (int r = 0; r < nr; ++r)
        s += FT[r * nth + c] * w[r];
      if (t >= 1)
        for (int i = 0; i < nx; ++i)
          s += VT[i + c * nx] * L[j * nx + i];
      TB[j * nth + c] += s;
    }
    ctx.sync();
  }

  // ---- initial: thbar += F0_x^T c_0 + F0_lam^T lambar_0 ----
  double *F0 = sm;
  th::copy(ctx, F0, a.kkt0fth + b * n0 * nth, n0 * nth);
  ctx.sync();
  for (int e = ctx.lane; e < R * nth; e += ctx.nl) {
    const int j = e / nth, c = e % nth;
    double s = 0.0;
    for (int i = 0; i < nx; ++i)
      s += F0[i * nth + c] * Cn[j * nx + i];
    if (a.clam0)
      for (int m = 0; m < nc0; ++m)
        s += F0[(nx + m) * nth + c] * a.clam0[rix(j, nc0) + m];
    a.theta_bar[rix(j, nth) + c] = TB[j * nth + c] + s;
  }
}

} // namespace ab2
