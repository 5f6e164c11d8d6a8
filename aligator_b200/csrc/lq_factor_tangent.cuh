// lq_factor_tangent.cuh -- forward mode of the backward recursion (ab2_gar_factor_tangent, include/aligator_b200/gar.h):
// the tangents of the factorisation FF, FB, VXX, VX, FFT, FBT along a tangent pdot of the problem records.  Plain C++
// apart from the execution context, so that the host emulation (tests/emu/factor_tangent_emu.cpp) compiles the same
// program.  It is the transpose of lq_factor_adjoint.cuh: <cbar, ydot> = <factor_adjoint(cbar), pdot>.
//
// The tangent recursion runs BACKWARD in time, as the sweep does: one work item (instance b) carries Vd, vd (the
// tangents of Vxx_{t+1}, vx_{t+1}) from the terminal knot to knot 0.  Per stage knot the forward quantities are
// recomputed from the record and the stored factor: V' = Vxx_{t+1}, X = [[K, k], [Z, z]], Shat = S + A^T V' B,
// v+ = vx_{t+1} + V' f, and M = [[R + B^T V' B, D^T], [D, -mu I]], factored again by Bunch-Kaufman from its lower
// triangle as resolve does.  With sym(P) = (P + P^T) / 2 and dotted blocks the tangent record:
//   products     vd+ = Vd' f + V' fd + vd',  Wd = Vd' B + V' Bd,  Td = Vd' A + 2 V' Ad
//                Shatd = Sd + Ad^T V' B + A^T Wd,  Rhatd = sym(Rd) + Bd^T V' B + B^T Wd,
//                Qhatd' = Qd + A^T Td   (sym(Qhatd') is the tangent of Qhat = Q + A^T V' A; only sym enters below)
//                rhatd = rd + Bd^T v+ + B^T vd+,  qhatd = qd + Ad^T v+ + A^T vd+
//   solve        [[Kd, kd], [Zd, zd]] = -M^-1 [[Rhatd K + Dd^T Z + Shatd^T, Rhatd k + Dd^T z + rhatd],
//                                               [Dd K + Cd,                 Dd k + dd               ]]
//   closed loop  Ahatd = Ad + Bd K + B Kd,  ad = fd + Bd k + B kd
//   value        Vxxd_t = sym(Qhatd' + Shatd K + Shat Kd + Cd^T Z + C^T Zd),
//                vxd_t = qhatd + Shatd k + Shat kd + Cd^T z + C^T zd
// and at the terminal knot (Z_N = C_N / mu, z_N = d_N / mu as stored in FBT, FFT):
//   Zd_N = Cd_N / mu,  zd_N = dd_N / mu,  Vxxd_N = sym(Qd_N + Cd_N^T Z_N + C_N^T Zd_N),  vxd_N = qd_N + Cd_N^T z_N +
//   C_N^T zd_N.
// The stored Q and R enter as sym(Qd), sym(Rd).  G0 and g0 do not enter the factorisation.
//
// Shared memory is the binding constraint at config 5: the item stages A, V', Vd' and Td (4 nx^2) and reads the dotted
// record blocks in place from global memory.  Vxxd_t is exactly symmetric: each entry is 0.5 (g_ij + g_ji) of the
// unsymmetrised sum g, formed by one lane.
//
// Work split: one item per instance, run by `nl` lanes that synchronise with ctx.sync() (one warp, or a whole CTA for
// items too large to share an SM).  Every entry of a result is summed by one lane in a fixed order, and the
// factorisation is resolve's, so the results do not depend on the lane count.
#pragma once

#include "lq_resolve.cuh"

namespace ab2 {

struct FactorTangentArgs {
  ResolveArgs fac;                  // records and factorisation: dims, stage .. G0, fb, fbT, Vxx, Vxx0, mueq, mueq_b
  const double *ff, *vx, *ffT;      // FF [batch][N][nu+nc+nx], VX [batch][N+1][nx], FFT [batch][nct]
  const double *d_stage, *d_term;   // tangent records in the problem's layouts, logical knot order; null = zero
  // tangents in ab2_gar_get's layouts (vxx full column-major [batch][N+1][nx*nx]); null = not written
  double *o_ff, *o_fb, *o_vxx, *o_vx, *o_fft, *o_fbt;
};

// doubles of shared memory one item uses: Vd, V', A, Td (nx^2); B, W = V'B, Wd, Shat, Shatd (nx nu); Rhatd (nu^2);
// C; [K; Z]; the solve P (n (nx + 1)); M and pivots; [k; z]; vd, f, v+, vd+
AB2_RS_HD int factor_tangent_item_doubles(int nx, int nu, int nc) {
  const int n = nu + nc;
  const int d = 4 * nx * nx + 5 * nx * nu + nu * nu + nc * nx + 4 * nx + n * (2 * nx + n + 3);
  return (d + 1) & ~1;
}

template <class Ctx>
AB2_RS_HD void factor_tangent_item(const FactorTangentArgs &a, const Ctx &ctx, double *sm, long b) {
  const ResolveArgs &r = a.fac;
  const int nx = r.nx, nu = r.nu, nc = r.nc, nct = r.nct, N = r.N;
  const int n = nu + nc, nr = n + nx, m = nx + 1;
  const double mu = r.mueq_b ? r.mueq_b[b] : r.mueq;
  double *Vd = sm, *Vp = Vd + nx * nx, *Am = Vp + nx * nx, *Td = Am + nx * nx;
  double *Bm = Td + nx * nx, *W = Bm + nx * nu, *Wd = W + nx * nu, *Sh = Wd + nx * nu, *Shd = Sh + nx * nu;
  double *Rd = Shd + nx * nu, *Cm = Rd + nu * nu, *KZ = Cm + nc * nx, *P = KZ + n * nx, *M = P + n * m;
  double *piv = M + n * n, *kz = piv + n, *vd = kz + n, *f = vd + nx, *vp = f + nx, *vdp = vp + nx;
  // all matrices column-major: Vd, Vp, Am, Td nx x nx; Bm, W, Wd, Sh, Shd nx x nu; Rd nu x nu; Cm nc x nx;
  // KZ = [K; Z] n x nx; P n x (nx + 1); M n x n

  // ---- terminal knot: record [Q | q | C | d] ----
  {
    const double *rec = r.term + b * r.trec, *CN = rec + nx * nx + nx;
    const double *ZN = r.fbT + b * nct * nx, *zN = a.ffT + b * nct;
    const double *dt = a.d_term ? a.d_term + b * r.trec : nullptr;
    const double *dC = dt ? dt + nx * nx + nx : nullptr, *dd = dC ? dC + nct * nx : nullptr;
    // g(p, q) = Qd_N + Cd_N^T Z_N + C_N^T Zd_N
    const auto g = [&](int p, int q) {
      double x = dt ? dt[p + q * nx] : 0.0, y = 0.0, z = 0.0;
      if (dC)
        for (int c = 0; c < nct; ++c) {
          y += dC[c + p * nct] * ZN[c * nx + q];
          z += CN[c + p * nct] * (dC[c + q * nct] / mu);
        }
      return (x + y) + z;
    };
    for (int e = ctx.lane; e < nx * nx; e += ctx.nl) {
      const int i = e % nx, j = e / nx;
      Vd[e] = 0.5 * (g(i, j) + g(j, i));
      if (a.o_vxx)
        a.o_vxx[(b * (N + 1) + N) * nx * nx + e] = Vd[e];
    }
    for (int i = ctx.lane; i < nx; i += ctx.nl) {
      double x = dt ? dt[nx * nx + i] : 0.0, y = 0.0, z = 0.0;
      if (dC)
        for (int c = 0; c < nct; ++c) {
          y += dC[c + i * nct] * zN[c];
          z += CN[c + i * nct] * (dd[c] / mu);
        }
      vd[i] = (x + y) + z;
      if (a.o_vx)
        a.o_vx[(b * (N + 1) + N) * nx + i] = vd[i];
    }
    if (a.o_fbt)
      for (int e = ctx.lane; e < nct * nx; e += ctx.nl) { // row-major: Zd_N[c][i] = Cd_N(c, i) / mu
        const int c = e / nx, i = e % nx;
        a.o_fbt[b * nct * nx + e] = dC ? dC[c + i * nct] / mu : 0.0;
      }
    if (a.o_fft)
      for (int c = ctx.lane; c < nct; c += ctx.nl)
        a.o_fft[b * nct + c] = dd ? dd[c] / mu : 0.0;
    ctx.sync();
  }

  for (int t = N - 1; t >= 0; --t) {
    const double *rec = r.stage + ((long)b * N + (t + r.stage_head >= N ? t + r.stage_head - N : t + r.stage_head)) * r.srec;
    // stage record [A | B | f | Q | S | R | q | r | C | D | d]
    const long oB = nx * nx, of = oB + nx * nu, oQ = of + nx, oS = oQ + nx * nx, oR = oS + nx * nu, oq = oR + nu * nu,
               orr = oq + nx, oC = orr + nu, oD = oC + nc * nx, od = oD + nc * nu;
    const double *ds = a.d_stage ? a.d_stage + ((long)b * N + t) * r.srec : nullptr; // the dotted record, read in place
    const double *fbk = r.fb + (b * N + t) * (long)nr * nx, *ffk = a.ff + (b * N + t) * (long)nr;

    // 1. stage V', A, B, f, C, [K; Z], [k; z]
    rs::load_v(r, ctx, b, t + 1, Vp);
    for (int e = ctx.lane; e < nx * nx; e += ctx.nl)
      Am[e] = rec[e];
    for (int e = ctx.lane; e < nx * nu; e += ctx.nl)
      Bm[e] = rec[oB + e];
    for (int e = ctx.lane; e < nc * nx; e += ctx.nl)
      Cm[e] = rec[oC + e];
    for (int e = ctx.lane; e < n * nx; e += ctx.nl) {
      const int i = e % n, j = e / n;
      KZ[e] = fbk[i * nx + j];
    }
    for (int i = ctx.lane; i < n; i += ctx.nl)
      kz[i] = ffk[i];
    for (int i = ctx.lane; i < nx; i += ctx.nl)
      f[i] = rec[of + i];
    ctx.sync();
    // 2. Td = Vd' A + 2 V' Ad, Wd = Vd' B + V' Bd, W = V' B; v+ = vx_{t+1} + V' f, vd+ = (vd' + Vd' f) + V' fd
    for (int e = ctx.lane; e < nx * (nx + 2 * nu); e += ctx.nl) {
      const int i = e % nx, c = e / nx;
      double s = 0.0, w = 0.0;
      if (c < nx) {
        for (int k = 0; k < nx; ++k)
          s += Vd[i + k * nx] * Am[k + c * nx];
        if (ds)
          for (int k = 0; k < nx; ++k)
            w += Vp[i + k * nx] * ds[k + c * nx];
        Td[e] = s + 2.0 * w;
      } else if (c < nx + nu) {
        const int u = c - nx;
        for (int k = 0; k < nx; ++k)
          s += Vd[i + k * nx] * Bm[k + u * nx];
        if (ds)
          for (int k = 0; k < nx; ++k)
            w += Vp[i + k * nx] * ds[oB + k + u * nx];
        Wd[i + u * nx] = s + w;
      } else {
        const int u = c - nx - nu;
        for (int k = 0; k < nx; ++k)
          s += Vp[i + k * nx] * Bm[k + u * nx];
        W[i + u * nx] = s;
      }
    }
    for (int i = ctx.lane; i < nx; i += ctx.nl) {
      double s = 0.0, sd = 0.0, w = 0.0;
      for (int k = 0; k < nx; ++k) {
        s += Vp[i + k * nx] * f[k];
        sd += Vd[i + k * nx] * f[k];
      }
      if (ds)
        for (int k = 0; k < nx; ++k)
          w += Vp[i + k * nx] * ds[of + k];
      vp[i] = a.vx[(b * (N + 1) + t + 1) * nx + i] + s;
      vdp[i] = (vd[i] + sd) + w;
    }
    ctx.sync();
    // 3. Vd <- Qhatd' = Qd + A^T Td; Shat = S + A^T W; Shatd = (Sd + Ad^T W) + A^T Wd;
    //    Rhatd = (sym(Rd) + Bd^T W) + B^T Wd; M (lower) = [[R + B^T W, .], [D, -mu I]]; vd <- qhatd
    for (int e = ctx.lane; e < nx * nx; e += ctx.nl) {
      const int i = e % nx, j = e / nx;
      double s = 0.0;
      for (int k = 0; k < nx; ++k)
        s += Am[k + i * nx] * Td[k + j * nx];
      Vd[e] = (ds ? ds[oQ + e] : 0.0) + s;
    }
    for (int e = ctx.lane; e < nx * nu; e += ctx.nl) {
      const int i = e % nx, c = e / nx;
      double s = 0.0, sd = 0.0, w = 0.0;
      for (int k = 0; k < nx; ++k) {
        s += Am[k + i * nx] * W[k + c * nx];
        w += Am[k + i * nx] * Wd[k + c * nx];
      }
      if (ds)
        for (int k = 0; k < nx; ++k)
          sd += ds[k + i * nx] * W[k + c * nx];
      Sh[e] = rec[oS + e] + s;
      Shd[e] = ((ds ? ds[oS + e] : 0.0) + sd) + w;
    }
    for (int e = ctx.lane; e < nu * nu; e += ctx.nl) {
      const int i = e % nu, j = e / nu;
      double s = 0.0, w = 0.0;
      if (ds)
        for (int k = 0; k < nx; ++k)
          s += ds[oB + k + i * nx] * W[k + j * nx];
      for (int k = 0; k < nx; ++k)
        w += Bm[k + i * nx] * Wd[k + j * nx];
      Rd[e] = ((ds ? 0.5 * (ds[oR + e] + ds[oR + j + i * nu]) : 0.0) + s) + w;
    }
    for (int e = ctx.lane; e < n * n; e += ctx.nl) {
      const int i = e % n, j = e / n;
      if (i < j)
        continue;
      double v;
      if (i < nu) {
        double s = 0.0;
        for (int k = 0; k < nx; ++k)
          s += Bm[k + i * nx] * W[k + j * nx];
        v = rec[oR + i + j * nu] + s;
      } else if (j < nu) {
        v = rec[oD + (i - nu) + j * nc];
      } else {
        v = i == j ? -mu : 0.0;
      }
      M[e] = v;
    }
    for (int i = ctx.lane; i < nx; i += ctx.nl) {
      double s = 0.0, w = 0.0;
      if (ds)
        for (int k = 0; k < nx; ++k)
          s += ds[k + i * nx] * vp[k];
      for (int k = 0; k < nx; ++k)
        w += Am[k + i * nx] * vdp[k];
      vd[i] = ((ds ? ds[oq + i] : 0.0) + s) + w;
    }
    ctx.sync();
    // 4. P = [[Rhatd K + Dd^T Z + Shatd^T, Rhatd k + Dd^T z + rhatd], [Dd K + Cd, Dd k + dd]]; factor M; P <- -M^-1 P
    for (int e = ctx.lane; e < n * m; e += ctx.nl) {
      const int i = e % n, j = e / n;
      const double *X = j < nx ? KZ + j * n : kz; // column j of [[K, k], [Z, z]]
      double s = 0.0, w = 0.0, h;
      if (i < nu) {
        for (int c = 0; c < nu; ++c)
          s += Rd[i + c * nu] * X[c];
        if (ds)
          for (int l = 0; l < nc; ++l)
            w += ds[oD + l + i * nc] * X[nu + l];
        if (j < nx) {
          h = Shd[j + i * nx];
        } else { // rhatd = (rd + Bd^T v+) + B^T vd+
          double y = 0.0, z = 0.0;
          if (ds)
            for (int k = 0; k < nx; ++k)
              y += ds[oB + k + i * nx] * vp[k];
          for (int k = 0; k < nx; ++k)
            z += Bm[k + i * nx] * vdp[k];
          h = ((ds ? ds[orr + i] : 0.0) + y) + z;
        }
      } else {
        const int l = i - nu;
        if (ds)
          for (int c = 0; c < nu; ++c)
            s += ds[oD + l + c * nc] * X[c];
        h = ds ? (j < nx ? ds[oC + l + j * nc] : ds[od + l]) : 0.0;
      }
      P[e] = (s + w) + h;
    }
    ctx.sync();
    rs::bk_factor(ctx, M, piv, n);
    for (int j = ctx.lane; j < m; j += ctx.nl) {
      rs::bk_solve(M, piv, n, P + j * n);
      for (int i = 0; i < n; ++i)
        P[i + j * n] = -P[i + j * n];
    }
    ctx.sync();
    // 5. outputs: FB rows [Kd; Zd; Ahatd], FF [kd; zd; ad]; Td <- Vxxd_t = sym(g), vd <- vxd_t
    if (a.o_fb) {
      double *o = a.o_fb + (b * N + t) * (long)nr * nx;
      for (int e = ctx.lane; e < nr * nx; e += ctx.nl) { // row-major
        const int i = e / nx, j = e % nx;
        if (i < n) {
          o[e] = P[i + j * n];
        } else { // Ahatd = (Ad + Bd K) + B Kd
          const int p = i - n;
          double s = 0.0, w = 0.0;
          if (ds)
            for (int c = 0; c < nu; ++c)
              s += ds[oB + p + c * nx] * KZ[c + j * n];
          for (int c = 0; c < nu; ++c)
            w += Bm[p + c * nx] * P[c + j * n];
          o[e] = ((ds ? ds[p + j * nx] : 0.0) + s) + w;
        }
      }
    }
    if (a.o_ff) {
      double *o = a.o_ff + (b * N + t) * (long)nr;
      for (int i = ctx.lane; i < nr; i += ctx.nl) {
        if (i < n) {
          o[i] = P[i + nx * n];
        } else { // ad = (fd + Bd k) + B kd
          const int p = i - n;
          double s = 0.0, w = 0.0;
          if (ds)
            for (int c = 0; c < nu; ++c)
              s += ds[oB + p + c * nx] * kz[c];
          for (int c = 0; c < nu; ++c)
            w += Bm[p + c * nx] * P[c + nx * n];
          o[i] = ((ds ? ds[of + p] : 0.0) + s) + w;
        }
      }
    }
    // g(p, q) = Qhatd' + Shatd K + Shat Kd + Cd^T Z + C^T Zd
    const auto g = [&](int p, int q) {
      double x = 0.0, y = 0.0, z = 0.0, w = 0.0;
      for (int c = 0; c < nu; ++c) {
        x += Shd[p + c * nx] * KZ[c + q * n];
        y += Sh[p + c * nx] * P[c + q * n];
      }
      if (ds)
        for (int l = 0; l < nc; ++l)
          z += ds[oC + l + p * nc] * KZ[nu + l + q * n];
      for (int l = 0; l < nc; ++l)
        w += Cm[l + p * nc] * P[nu + l + q * n];
      return (((Vd[p + q * nx] + x) + y) + z) + w;
    };
    for (int e = ctx.lane; e < nx * nx; e += ctx.nl) {
      const int i = e % nx, j = e / nx;
      Td[e] = 0.5 * (g(i, j) + g(j, i));
      if (a.o_vxx)
        a.o_vxx[(b * (N + 1) + t) * nx * nx + e] = Td[e];
    }
    for (int i = ctx.lane; i < nx; i += ctx.nl) {
      double x = 0.0, y = 0.0, z = 0.0, w = 0.0;
      for (int c = 0; c < nu; ++c) {
        x += Shd[i + c * nx] * kz[c];
        y += Sh[i + c * nx] * P[c + nx * n];
      }
      if (ds)
        for (int l = 0; l < nc; ++l)
          z += ds[oC + l + i * nc] * kz[nu + l];
      for (int l = 0; l < nc; ++l)
        w += Cm[l + i * nc] * P[nu + l + nx * n];
      vd[i] = (((vd[i] + x) + y) + z) + w;
      if (a.o_vx)
        a.o_vx[(b * (N + 1) + t) * nx + i] = vd[i];
    }
    ctx.sync();
    double *tmp = Vd; // the carry Vd' of knot t - 1 is Td
    Vd = Td;
    Td = tmp;
  }
}

} // namespace ab2
