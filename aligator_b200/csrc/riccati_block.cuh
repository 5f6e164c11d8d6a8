// riccati_block.cuh -- the sweep for ARBITRARY (run-time) dimensions: one CTA per
// instance, every matrix in shared memory, the dense products of the knot step tiled
// 8x8x4 on the FP64 tensor cores (DMMA) and spread over the CTA's warps.
//
// Serves the shapes the warp-per-instance kernels of riccati_group.cuh cannot hold:
// large states (BASELINE config 5: nx = 56, nu = 22), constrained knots with
// nu + nc > 32 rows in the reduced KKT matrix, and any (nx, nu, nc) that was not
// instantiated at compile time.  Same mathematics, same reference citations
// (gar/riccati-kernel.hxx:105-377, core/bunchkaufman.hpp) and the same logical column
// order [A | f | B] as stage_loop_mma; the Bunch-Kaufman factorisation is the
// cooperative bk_factor_group with one THREAD per matrix row.
//
// Compiles for the host as well (tests/emu/block_emu.cpp): a CTA is T std::threads.
//
// Ctx: tid, nthreads, warp, lane, nwarps; sync() = CTA barrier; mma(d, a, b) = one
// warp-wide m8n8k4 f64 MMA; issue_copy(part, dst, src, nd) / wait_copy(part) = TMA bulk
// copy global -> shared completing on mbarrier `part` (issued by one thread, waited by all).
#pragma once

#include "riccati_group.cuh"

namespace ab2 {

struct BlockDims {
  static constexpr int static_nk = 0; // run-time dimensions: no register-resident factorisation
  int nx, nu, nc; // stage knots
  int nk, nr, nj, mtx, kt, nt, nt2, kt2, njp;
  int off_b, off_f, off_q, off_s, off_r, off_qv, off_rv, off_c, off_d, off_dv, srec_pad;
  int split; // [0, split) = [A B f] (live until the closing products), [split, srec_pad) = the rest
  int vs, vrows, sw, wrows, sh, sx, xrows;
  int s_rec, s_vn, s_vxn, s_w, s_x, s_kk, s_y, s_h, s_kkt, s_dd, s_sd, s_int, s_end; // doubles
  int fwd_ring, fwd_slot, slack;
  // parametric terms (nth > 0): record offsets [Gx | Gu | Gv | Gth | gamma] and the theta workspace
  int nth, rec_nth, off_gx, off_gu, off_gv, off_gth, off_gam;
  int s_th; // start of the theta workspace (behind everything else, incl. the initial-stage overlay)
};

AB2_HD constexpr int blk_ev(int x) { return (x + 1) & ~1; }
AB2_HD constexpr int blk_fstride(int n) { // smallest stride >= n that is 4 or 12 mod 16
  int s = n;
  while (s % 16 != 4 && s % 16 != 12)
    ++s;
  return s;
}
AB2_HD constexpr int blk_s8(int n) { // smallest stride >= n that is 8 mod 16
  int s = n;
  while (s % 16 != 8)
    ++s;
  return s;
}

// Layout shared by the host (sizing the launch) and the device.
// nth: parameter dimension of the value function (workspace); rec_nth: parameter blocks carried
// by the knot RECORDS (-1 = nth).  Leg mode (ParallelRiccatiSolver, gar/parallel-solver.hxx) has
// nth = nx with plain records: the parameterisation of a leg is implicit (Gx = A^T, Gu = B^T,
// gamma = f on the leg's last knot, zero elsewhere, :136-147).
AB2_HD constexpr BlockDims make_block_dims(int nx, int nu, int nc, int nc0, int nth = 0, int rec_nth = -1) {
  BlockDims d{};
  d.nth = nth;
  if (rec_nth < 0)
    rec_nth = nth;
  d.rec_nth = rec_nth;
  d.nx = nx;
  d.nu = nu;
  d.nc = nc;
  d.nk = nu + nc;
  d.nr = nu + nc + nx;
  d.nj = nx + 1 + nu;
  d.mtx = (nx + 7) / 8;
  d.kt = (nx + 3) / 4;
  d.nt = (d.nj + 7) / 8;
  d.nt2 = (nx + 1 + 7) / 8;
  d.kt2 = (d.nk + 3) / 4;
  d.njp = 8 * d.nt;
  const StageOffsets so = stage_offsets(nx, nu, nc);
  const TailOffsets tail = stage_tail(so, nx, nu, nc, rec_nth);
  d.off_b = so.B;
  d.off_f = so.f;
  d.off_q = so.Q;
  d.off_s = so.S;
  d.off_r = so.R;
  d.off_qv = so.q;
  d.off_rv = so.r;
  d.off_c = so.C;
  d.off_d = so.D;
  d.off_dv = so.d;
  d.off_gx = tail.Gx;
  d.off_gu = tail.Gu;
  d.off_gv = tail.Gv;
  d.off_gth = tail.Gth;
  d.off_gam = tail.gamma;
  d.srec_pad = stage_pad(tail.end);
  // (parametric knots read [Gx .. gamma] at the end of the step: no early refill of the tail)
  d.split = (d.off_q % 2 == 0 && rec_nth == 0) ? d.off_q : d.srec_pad;
  d.vs = blk_fstride(4 * d.kt);
  d.vrows = 8 * d.mtx;
  d.sw = blk_fstride(d.njp); // (W is read as the B operand of (2): row stride 4 or 12 mod 16, conflict-free)
  d.wrows = 4 * d.kt;
  d.sh = blk_s8(d.njp);
  d.sx = blk_fstride(8 * d.nt2 + nth); // columns [K | k | theta columns nx+1..nx+nth]
  d.xrows = 4 * d.kt2;
  int o = 0;
  d.s_rec = o;
  d.slack = blk_ev(4 * d.kt + 8); // zeroed: the "column" every padding column of M points at
  o += d.srec_pad + d.slack;
  d.s_vn = o;
  o += blk_ev(d.vrows * d.vs);
  d.s_vxn = o;
  o += blk_ev(nx);
  d.s_h = o;
  o += blk_ev(d.njp * d.sh);
  const int xsz = blk_ev(d.xrows * d.sx);
  d.s_w = o; // W; once consumed, the same space holds X, KK and the solve scratch Y
  d.s_x = o;
  d.s_kk = o + xsz;
  {
    // the solve scratch Y lives in the control rows of Hs (dead once X and the KKT matrix
    // are built) when it fits there, else behind KK
    const bool y_in_h = xsz <= (d.njp - nx - 1) * d.sh;
    d.s_y = y_in_h ? d.s_h + (nx + 1) * d.sh : o + 2 * xsz;
    const int a = blk_ev(d.wrows * d.sw), b = (y_in_h ? 2 : 3) * xsz;
    o += a > b ? a : b;
  }
  d.s_kkt = o;
  o += blk_ev(d.nk * d.nk);
  d.s_dd = o;
  o += blk_ev(d.nk);
  d.s_sd = o;
  o += blk_ev(d.nk);
  d.s_int = o;
  o += blk_ev(d.nk + 1);
  // the initial-stage saddle system overlays everything: K0 n0*n0, 5 vectors, 2*n0 ints
  const int n0 = nx + nc0;
  const int k0 = n0 * n0 + 6 * n0 + 2;
  d.s_end = blk_ev(o > k0 ? o : k0);
  d.s_th = d.s_end;
  if (nth > 0) // theta workspace: Vxt', Vtt', vt' (double-buffered), Gxhat, 3 x the initial-stage theta columns
    d.s_end += blk_ev(2 * nx * nth) + blk_ev(2 * nth * nth) + blk_ev(2 * nth) + blk_ev(nx * nth) + 3 * blk_ev(n0 * nth);
  // forward: ring of fb records + two state vectors
  d.fwd_slot = blk_ev(d.nr * nx) + 2; // an odd-sized record is fetched from the aligned double before it
  int ring = (d.s_end - 2 * blk_ev(nx)) / d.fwd_slot;
  if (ring < 1) {
    ring = 1;
    d.s_end = d.fwd_slot + 2 * blk_ev(nx);
  }
  d.fwd_ring = ring > 8 ? 8 : ring;
  return d;
}

// The same layout with every field a compile-time constant: a specialisation of the kernel
// for one shape (loops unroll, addresses fold) behind the same code.
template <int NX, int NU, int NC, int NC0> struct StaticBlockDims {
  static constexpr BlockDims v = make_block_dims(NX, NU, NC, NC0);
  // KKT size known at compile time and <= 32 rows: the LDL^T runs from the registers of one warp
  static constexpr int static_nk = (NC == 0 && NU <= 32) ? NU : 0;
#define AB2_SD(f) static constexpr int f = v.f;
  AB2_SD(nx) AB2_SD(nu) AB2_SD(nc) AB2_SD(nk) AB2_SD(nr) AB2_SD(nj) AB2_SD(mtx) AB2_SD(kt) AB2_SD(nt) AB2_SD(nt2)
  AB2_SD(kt2) AB2_SD(njp) AB2_SD(off_b) AB2_SD(off_f) AB2_SD(off_q) AB2_SD(off_s) AB2_SD(off_r) AB2_SD(off_qv)
  AB2_SD(off_rv) AB2_SD(off_c) AB2_SD(off_d) AB2_SD(off_dv) AB2_SD(srec_pad) AB2_SD(split) AB2_SD(vs) AB2_SD(vrows)
  AB2_SD(sw) AB2_SD(wrows) AB2_SD(sh) AB2_SD(sx) AB2_SD(xrows) AB2_SD(s_rec) AB2_SD(s_vn) AB2_SD(s_vxn) AB2_SD(s_w)
  AB2_SD(s_x) AB2_SD(s_kk) AB2_SD(s_y) AB2_SD(s_h) AB2_SD(s_kkt) AB2_SD(s_dd) AB2_SD(s_sd) AB2_SD(s_int) AB2_SD(s_end)
  AB2_SD(fwd_ring) AB2_SD(fwd_slot) AB2_SD(slack) AB2_SD(nth) AB2_SD(off_gx) AB2_SD(off_gu) AB2_SD(off_gv)
  AB2_SD(off_gth) AB2_SD(off_gam) AB2_SD(s_th) AB2_SD(rec_nth)
#undef AB2_SD
};

template <class D> AB2_D int blk_col_offset(const D &d, int jp) { // logical column jp of [A | f | B]
  if (jp < d.nx)
    return jp * d.nx;
  if (jp == d.nx)
    return d.off_f;
  if (jp <= d.nx + d.nu)
    return d.off_b + (jp - d.nx - 1) * d.nx;
  return d.srec_pad; // padding column: the zeroed slack behind the record
}
template <class D> AB2_D int blk_h0_offset(const D &d, int ip, int jp) { // -1 = structural zero
  const int nx = d.nx, nu = d.nu;
  const int ti = ip < nx ? 0 : (ip == nx ? 1 : (ip <= nx + nu ? 2 : 3));
  const int tj = jp < nx ? 0 : (jp == nx ? 1 : (jp <= nx + nu ? 2 : 3));
  const int ci = ip - nx - 1, cj = jp - nx - 1;
  if (ti == 0 && tj == 0)
    return d.off_q + jp * nx + ip;
  if (ti == 0 && tj == 2)
    return d.off_s + cj * nx + ip;
  if (ti == 2 && tj == 0)
    return d.off_s + ci * nx + jp;
  if (ti == 2 && tj == 2)
    return d.off_r + cj * nu + ci;
  if (ti == 0 && tj == 1)
    return d.off_qv + ip;
  if (ti == 2 && tj == 1)
    return d.off_rv + ci;
  return -1;
}

// The whole CTA seen as one "group" by the cooperative Bunch-Kaufman routines
// (one thread per matrix row, CTA-wide barrier).
template <class Ctx> struct CtaAsGroup {
  Ctx &c;
  int lane;
  int nthreads; // participating threads (a multiple of 32): barrier over those warps only
  AB2_D void sync() { c.sync_sub(nthreads); }
};

// Per-thread solve of one right-hand-side column with the factor left by
// bk_factor_group (run-time n; same sequence as bk_solve_column: interchanges, unit-lower
// solve, D^-1, unit-upper solve, inverse interchanges).  Both triangular solves run in
// dot-product form -- x_i = b_i - sum_c L(i,c) x_c -- so the loads of one row pipeline
// (no store in between) and the code stays small (a fully unrolled register version
// stalls on instruction fetch).  rhs/work/sol: column pointers, rows `stride` apart; the
// result is -(KKT^-1 rhs).
AB2_D void bk_solve_column_rt(const double *a, const int n, const double *dd, const double *sd,
                              const int *perm, const int *kind, const double *rhs, double *work,
                              double *sol, const int stride, const bool negate = true) {
  for (int i = 0; i < n; ++i)
    work[i * stride] = rhs[perm[i] * stride];
  for (int i = 1; i < n; ++i) { // forward: unit lower, row i of L against x_0..x_{i-1}
    double s0 = work[i * stride], s1 = 0.0;
    const double *li = a + i;   // L(i, c) = li[c * n]
    int c = 0;
    for (; c + 4 <= i; c += 4) { // four loads of each operand in flight, two accumulation chains
      const double l0 = li[c * n], l1 = li[(c + 1) * n], l2 = li[(c + 2) * n], l3 = li[(c + 3) * n];
      const double x0 = work[c * stride], x1 = work[(c + 1) * stride], x2 = work[(c + 2) * stride],
                   x3 = work[(c + 3) * stride];
      s0 -= l0 * x0;
      s1 -= l1 * x1;
      s0 -= l2 * x2;
      s1 -= l3 * x3;
    }
    for (; c < i; ++c)
      s0 -= li[c * n] * work[c * stride];
    work[i * stride] = s0 + s1;
  }
  for (int k = 0; k < n; ++k) {
    const int kd = kind[k];
    if (kd == 0) {
      work[k * stride] *= dd[k];
    } else if (kd == 1 && k + 1 < n) {
      const double xk = work[k * stride], xk1 = work[(k + 1) * stride], s = sd[k];
      work[k * stride] = xk * dd[k] + xk1 * s;
      work[(k + 1) * stride] = xk1 * dd[k + 1] + xk * s;
    }
  }
  for (int c = n - 2; c >= 0; --c) { // backward: unit upper (L^T), column c of L against x_{c+1}..x_{n-1}
    double s0 = work[c * stride], s1 = 0.0;
    const double *lc = a + c * n; // L(i, c) = lc[i]
    int i = c + 1;
    for (; i + 4 <= n; i += 4) {
      const double l0 = lc[i], l1 = lc[i + 1], l2 = lc[i + 2], l3 = lc[i + 3];
      const double x0 = work[i * stride], x1 = work[(i + 1) * stride], x2 = work[(i + 2) * stride],
                   x3 = work[(i + 3) * stride];
      s0 -= l0 * x0;
      s1 -= l1 * x1;
      s0 -= l2 * x2;
      s1 -= l3 * x3;
    }
    for (; i < n; ++i)
      s0 -= lc[i] * work[i * stride];
    work[c * stride] = s0 + s1;
  }
  for (int i = 0; i < n; ++i)
    sol[perm[i] * stride] = negate ? -work[i * stride] : work[i * stride];
}

// LDL^T of a matrix on which every pivot test of the Bunch-Kaufman algorithm picks the 1x1
// pivot in place (|a_kk| >= alpha * colmax, core/bunchkaufman.hpp:61; the SPD Rhat of an
// unconstrained knot) -- the same arithmetic as the general algorithm on that path (and as
// FastFactor of the warp-per-instance kernel), run by ONE warp with lane = row: the column
// test is a vote, the pivot row travels by shuffle, no scan, no barrier between warps.
// Leaves the factor in the format of bk_factor_group (identity interchanges).  Returns false
// at the first pivot test that fails; the matrix is then partly overwritten (the caller
// restores its copy and runs the general algorithm).
template <class Ctx>
AB2_D bool ldlt_fast_warp(Ctx &ctx, double *a, const int n, double *dd, double *sd, int *perm, int *kind) {
  const double alpha = 0.6403882032022076; // (1+sqrt(17))/8
  const int lane = ctx.lane;
  for (int k = 0; k < n; ++k) {
    ctx.wsync(); // column k is final
    const double akk = a[k + k * n];
    const bool below = lane > k && lane < n;
    const double my = below ? a[lane + k * n] : 0.0;
    const bool ok = (fabs(my) * alpha <= fabs(akk)) && (fabs(akk) > 0.0);
    if (!ctx.all(ok))
      return false;
    const double d = 1.0 / akk;
    if (lane == k) {
      dd[k] = d;
      sd[k] = 0.0;
      kind[k] = 0;
      perm[k] = k;
    }
    // trailing rows: a_ij -= (a_jk d) a_ik, i >= j.  Four columns per round: the shuffles and
    // the loads of a round are independent, so a lone warp overlaps their latencies.
    int j = k + 1;
    for (; j + 4 <= n; j += 4) {
      const double m0 = ctx.shfl(my, j), m1 = ctx.shfl(my, j + 1), m2 = ctx.shfl(my, j + 2),
                   m3 = ctx.shfl(my, j + 3);
      const bool in = lane < n;
      double *p = a + lane + j * n;
      const double r0 = in ? p[0] : 0.0, r1 = in ? p[n] : 0.0, r2 = in ? p[2 * n] : 0.0, r3 = in ? p[3 * n] : 0.0;
      if (in && lane >= j)
        p[0] = r0 - (m0 * d) * my;
      if (in && lane >= j + 1)
        p[n] = r1 - (m1 * d) * my;
      if (in && lane >= j + 2)
        p[2 * n] = r2 - (m2 * d) * my;
      if (in && lane >= j + 3)
        p[3 * n] = r3 - (m3 * d) * my;
    }
    for (; j < n; ++j) {
      const double mj = ctx.shfl(my, j);
      if (lane >= j && lane < n)
        a[lane + j * n] -= (mj * d) * my;
    }
    if (below)
      a[lane + k * n] = my * d;
  }
  ctx.wsync();
  return true;
}

// phase clocks (profiling aid): thread 0 of the CTA that owns instance 0 accumulates clock64() deltas
#if defined(__CUDA_ARCH__)
#define AB2_CLK_INIT long long clk_t0 = (p.clk && inst == 0 && tid == 0) ? clock64() : 0
#define AB2_CLK(ph)                                                        \
  do {                                                                     \
    if (p.clk && inst == 0 && tid == 0) {                                  \
      const long long now_ = clock64();                                    \
      p.clk[ph] += now_ - clk_t0;                                          \
      clk_t0 = now_;                                                       \
    }                                                                      \
  } while (0)
#else
#define AB2_CLK_INIT (void)0
#define AB2_CLK(ph) (void)0
#endif

// LDL^T by the WHOLE CTA of a matrix on which every pivot test of the Bunch-Kaufman algorithm picks
// the 1x1 pivot in place by its first test (|a_kk| >= alpha*colmax, core/bunchkaufman.hpp:61).  Same
// arithmetic as bk_factor_group / ldlt_fast_warp on that path, but one thread per ELEMENT of the
// trailing triangle instead of one lane per row: per column one barrier (which carries the vote),
// three loads, two flops and a store per thread, where the single-warp routine walks each row in
// rounds of four.  Matrix in shared memory (column-major, lda = n);
// leaves L / dd / sd / perm / kind in bk_factor_group's format.  Returns false at the first failing test
// (uniform over the CTA) with the matrix partly updated: the caller restores its copy.
template <class Ctx>
AB2_D bool ldlt_fast_cta(Ctx &ctx, double *a, const int n, double *dd, double *sd, int *perm, int *kind) {
  const double alpha = 0.6403882032022076; // (1+sqrt(17))/8
  const int tid = ctx.tid, lane = ctx.lane, warp = ctx.warp, NW = ctx.nwarps;
  // n <= 32.  Columns stay UNSCALED during the elimination (the update multiplies by d on the fly,
  // exactly the reference's (a_jk d) a_ik) and are scaled in one pass at the end.  ONE barrier per
  // column: warp 0, which produces the next pivot column, tests it from its registers (pivot by
  // shuffle) and the barrier carries that vote to the CTA.
  bool bad = false;
  if (warp == 0) { // test of column 0
    const double v = lane < n ? a[lane] : 0.0;
    const double piv = ctx.shfl(v, 0);
    bad = (lane >= 1 && lane < n && !(fabs(v) * alpha <= fabs(piv))) || (lane == 0 && !(fabs(piv) > 0.0));
  }
  if (ctx.sync_or(bad ? 1 : 0))
    return false;
  for (int k = 0; k < n; ++k) {
    const double akk = a[k + k * n];
    const double d = rcp_fast(akk); // (as FastFactor: within an ulp of 1/akk)
    if (tid == k) {
      dd[k] = d;
      sd[k] = 0.0;
      kind[k] = 0;
      perm[k] = k;
    }
    // trailing triangle i >= j > k: lane = row offset, the warps deal out the columns; every access
    // is a broadcast or unit-stride over the lanes
    const int m = n - k - 1;
    double mycol = 0.0; // warp 0: the new entry of column k+1 in this lane's row
    if (lane < m) {
      const int i = k + 1 + lane;
      const double aik = a[i + k * n];
      for (int jj = warp; jj <= lane; jj += NW) {
        const int j = k + 1 + jj;
        const double v = a[i + j * n] - (a[j + k * n] * d) * aik;
        a[i + j * n] = v;
        if (jj == 0)
          mycol = v;
      }
    }
    bad = false;
    if (warp == 0 && m > 0) { // pivot test of column k+1 (rows k+1+lane, lane < m; its pivot sits in lane 0)
      const double piv = ctx.shfl(mycol, 0);
      bad = (lane >= 1 && lane < m && !(fabs(mycol) * alpha <= fabs(piv))) || (lane == 0 && !(fabs(piv) > 0.0));
    }
    if (ctx.sync_or(bad ? 1 : 0))
      return false;
  }
  for (int e = tid; e < n * n; e += ctx.nthreads) { // L = unscaled columns times d_k
    const int i = e % n, kcol = e / n;
    if (i > kcol)
      a[e] *= dd[kcol];
  }
  ctx.sync();
  return true;
}

// The same factorisation by ONE warp with the row in REGISTERS (N compile-time, <= 32): lane = row;
// per column the pivot by shuffle, the test by a vote, then every later column of the row updated
// with the multiplier shuffled from its own row -- independent shuffles and FMAs, no shared-memory
// round trip and no CTA barrier inside the elimination (the CTA-wide version above spends ~740
// cycles per column at n = 28, most of it in its barrier).  Reads the lower triangle from `a`
// (column-major, lda = N), writes L / dd / sd / perm / kind in bk_factor_group's format.  Returns
// false at the first failing test WITHOUT having written anything.
template <int N, int K, class Ctx>
AB2_D bool ldlt_regs_col(Ctx &ctx, double (&r)[N], double &myd) { // column K, compile-time: static register indices
  const double alpha = 0.6403882032022076; // (1+sqrt(17))/8
  const int lane = ctx.lane;
  const double akk = ctx.shfl(r[K], K);
  const double my = (lane > K) ? r[K] : 0.0; // a(lane, K) below the diagonal
  const bool ok = (fabs(my) * alpha <= fabs(akk)) && (fabs(akk) > 0.0);
  if (!ctx.all(ok))
    return false;
  const double d = rcp_fast(akk);
  if (lane == K)
    myd = d;
  const double lk = my * d; // L(lane, K)
  AB2_UNROLL
  for (int j = K + 1; j < N; ++j) {
    const double ljk = ctx.shfl(lk, j); // L(j, K)
    if (lane >= j)
      r[j] -= ljk * my; // a_ij -= (a_jk d) a_ik
  }
  if (lane > K)
    r[K] = lk;
  return true;
}
template <int N, class Ctx, int... Ks>
AB2_D bool ldlt_regs_cols(Ctx &ctx, double (&r)[N], double &myd, std::integer_sequence<int, Ks...>) {
  return (ldlt_regs_col<N, Ks>(ctx, r, myd) && ...); // stops at the first failing pivot test
}
template <int N, class Ctx>
AB2_D bool ldlt_regs_warp(Ctx &ctx, double *a, double *dd, double *sd, int *perm, int *kind) {
  const int lane = ctx.lane;
  double r[N]; // row `lane`: r[j] = a(lane, j), j <= lane
  AB2_UNROLL
  for (int j = 0; j < N; ++j)
    r[j] = (lane < N && j <= lane) ? a[lane + j * N] : 0.0;
  double myd = 0.0;
  if (!ldlt_regs_cols<N>(ctx, r, myd, std::make_integer_sequence<int, N>{}))
    return false;
  if (lane < N) {
    AB2_UNROLL
    for (int j = 0; j < N; ++j)
      if (j < lane)
        a[lane + j * N] = r[j];
    dd[lane] = myd;
    sd[lane] = 0.0;
    kind[lane] = 0;
    perm[lane] = lane;
  }
  ctx.wsync();
  return true;
}

// Run-time n <= NP: the matrix is padded to NP with an identity block (pivots 1, nothing below them:
// the padding columns pass every test and change nothing), so the small KKT matrices of the run-time
// kernel (n <= 16) take the register path too instead of a CTA barrier per column.
template <int NP, class Ctx>
AB2_D bool ldlt_regs_warp_pad(Ctx &ctx, double *a, const int n, double *dd, double *sd, int *perm, int *kind) {
  const int lane = ctx.lane;
  double r[NP];
  AB2_UNROLL
  for (int j = 0; j < NP; ++j) {
    const double v = a[(lane < n && j <= lane) ? lane + j * n : 0];
    r[j] = (lane < n && j <= lane) ? v : (j == lane ? 1.0 : 0.0);
  }
  double myd = 0.0;
  if (!ldlt_regs_cols<NP>(ctx, r, myd, std::make_integer_sequence<int, NP>{}))
    return false;
  if (lane < n) {
    AB2_UNROLL
    for (int j = 0; j < NP; ++j)
      if (j < lane)
        a[lane + j * n] = r[j];
    dd[lane] = myd;
    sd[lane] = 0.0;
    kind[lane] = 0;
    perm[lane] = lane;
  }
  ctx.wsync();
  return true;
}

// [K k] = -(L D L^T)^-1 X for a factor with identity interchanges and 1x1 pivots (what ldlt_fast_cta
// leaves), n <= 32: one warp per chunk of 8 right-hand-side columns, lane = ROW, the 8 entries of the
// row in registers.  Per elimination column c the pivot entries travel by shuffle and L(lane, c) is
// read ONCE for all 8 columns (conflict-free: consecutive lanes, consecutive addresses); the 8
// chains are independent, so shuffle and FMA latencies overlap.  (The thread-per-column routine
// re-reads x from shared memory behind every store and, at n = 28 with 58 columns, keeps only two
// warps busy; this uses all the CTA's warps.)  Same substitutions in the same order as
// bunch_kaufman_solve_in_place on that path (core/bunchkaufman.hpp:472-504).
// X, K: nk x ncols, row r at r*sx.
template <class Ctx>
AB2_D void ldlt_solve_rows_warp(Ctx &ctx, const double *a, const int n, const double *dd, const double *X, double *K,
                                const int sx, const int ncols) {
  constexpr int CW = 8; // columns per chunk
  const int lane = ctx.lane;
  const bool in = lane < n;
  const int row = in ? lane : 0;
  const double myd = in ? dd[row] : 0.0;
  for (int ch = ctx.warp; ch * CW < ncols; ch += ctx.nwarps) {
    const int j0 = ch * CW;
    double x[CW];
    AB2_UNROLL
    for (int u = 0; u < CW; ++u)
      x[u] = (in && j0 + u < ncols) ? X[row * sx + j0 + u] : 0.0;
    for (int c = 0; c + 1 < n; ++c) { // unit lower, column-oriented
      const double l = (in && lane > c) ? a[row + c * n] : 0.0;
      AB2_UNROLL
      for (int u = 0; u < CW; ++u)
        x[u] -= l * ctx.shfl(x[u], c);
    }
    AB2_UNROLL
    for (int u = 0; u < CW; ++u)
      x[u] *= myd;
    for (int i = n - 1; i >= 1; --i) { // unit upper (L^T)
      const double l = (in && lane < i) ? a[i + row * n] : 0.0;
      AB2_UNROLL
      for (int u = 0; u < CW; ++u)
        x[u] -= l * ctx.shfl(x[u], i);
    }
    if (in) {
      AB2_UNROLL
      for (int u = 0; u < CW; ++u)
        if (j0 + u < ncols)
          K[row * sx + j0 + u] = -x[u];
    }
  }
}

constexpr int BLK_CH = 4; // n-tiles accumulated together by one warp (one work item)

// ---------------------------------------------------------------------------
// The sweep of one instance by one CTA.
// ---------------------------------------------------------------------------
// mu: where this instance's mu is read (ScalarMu / InstanceMu, riccati_group.cuh).
template <class Ctx, class D, class Mu = ScalarMu>
AB2_D void riccati_block_sweep(Ctx &ctx, const SweepParams &p, const D &d, const int inst,
                               double *__restrict__ sm, const int leg = 0, const Mu &mu = Mu()) {
  const int nx = d.nx, nu = d.nu, nc = d.nc, nk = d.nk, nr = d.nr;
  const int tid = ctx.tid, T = ctx.nthreads, warp = ctx.warp, lane = ctx.lane, NW = ctx.nwarps;
  const int g = lane >> 2, q = lane & 3;
  const int N = p.N, nct = p.nct, nc0 = p.nc0;
  // leg mode: this CTA owns knots [t_lo, t_hi) of the instance (gar/parallel-solver.hxx:150-164)
  const int NLEG = p.legs > 1 ? p.legs : 1;
  const bool legmode = NLEG > 1;
  const int t_lo = legmode ? leg_begin(N, leg, NLEG) : 0;
  const int t_hi = legmode ? leg_begin(N, leg + 1, NLEG) : N + 1;
  const bool last_leg = t_hi == N + 1; // the leg that holds the terminal knot (no parameters)

  double *rec = sm + d.s_rec;
  double *Vn = sm + d.s_vn;
  double *vxn = sm + d.s_vxn;
  double *Hs = sm + d.s_h;
  double *Wsm = sm + d.s_w;
  double *X = sm + d.s_x;
  double *KKs = sm + d.s_kk;
  double *Ys = sm + d.s_y;
  double *kkt = sm + d.s_kkt;
  double *dd = sm + d.s_dd;
  double *sd = sm + d.s_sd;
  int *perm = reinterpret_cast<int *>(sm + d.s_int);
  int *kind = perm + nk;

  const double *stage_b = p.stage + (size_t)inst * N * d.srec_pad;
  double *ff_b = p.ff + (size_t)inst * N * nr;
  double *fb_b = p.fb + (size_t)inst * N * nr * nx;
  double *Vxx_b = p.Vxx + (size_t)inst * (N + 1) * nx * nx;
  double *vx_b = p.vx + (size_t)inst * (N + 1) * nx;
  const int bk_threads = 32 * ((nk + 31) / 32); // warps that own rows of the KKT matrix
  CtaAsGroup<Ctx> grp{ctx, tid, bk_threads};
  // ---- parametric terms (nth > 0): workspace behind everything else ----
  const int nth = (legmode && last_leg) ? 0 : d.nth;
  double *th = sm + d.s_th;
  double *vxt2 = th;                                  // [2][nx*nth]  Vxt' (current / next), column-major
  double *vtt2 = vxt2 + blk_ev(2 * nx * nth);         // [2][nth*nth]
  double *vtv2 = vtt2 + blk_ev(2 * nth * nth);        // [2][nth]
  double *gxh = vtv2 + blk_ev(2 * nth);               // Gxhat nx x nth column-major
  const int thn = (nx + nc0) * nth;                   // the initial-stage solve of the theta columns
  double *trhs = gxh + blk_ev(nx * nth);              // right-hand sides [row][nth]
  double *twork = trhs + blk_ev(thn);
  double *tsol = twork + blk_ev(thn);
  int thcur = 0;                                      // which half of vxt2 / vtt2 / vtv2 holds V'
  double *fth_b = nth ? p.fth + (size_t)inst * N * nr * nth : nullptr;
  double *Vxt_b = nth ? p.Vxt + (size_t)inst * (N + 1) * nx * nth : nullptr;
  double *Vtt_b = nth ? p.Vtt + (size_t)inst * (N + 1) * nth * nth : nullptr;
  double *vt_b = nth ? p.vt + (size_t)inst * (N + 1) * nth : nullptr;
  const bool two_parts = d.split < d.srec_pad;

  if (p.do_bwd) {
    AB2_CLK_INIT;
    int st = ST_OK;
    int pv = 0; // pivot statistics (threads 0..bk_threads-1 all see the same decisions)
    const int t_first = last_leg ? N - 1 : t_hi - 1; // first stage knot of the (descending) loop
    if (t_first >= t_lo) {
      const double *src = stage_b + (size_t)stage_slot(p, t_first) * d.srec_pad;
      ctx.issue_copy(0, rec, src, d.split);
      if (two_parts)
        ctx.issue_copy(1, rec + d.split, src + d.split, d.srec_pad - d.split);
    }
    for (int i = tid; i < d.vrows * d.vs; i += T)
      Vn[i] = 0.0;
    for (int i = tid; i < d.slack; i += T)
      rec[d.srec_pad + i] = 0.0; // the slack behind the record
    // W / X / KK / Y: padding entries are multiplied by structural zeros, so they must be finite
    for (int i = tid; i < d.s_kkt - d.s_w; i += T)
      Wsm[i] = 0.0;
    ctx.sync();
    if (!last_leg) {
      // A leg that ends on a stage knot: that knot is the leg's terminal knot WITH controls
      // (riccati-kernel.hxx:151-172, 185-192), parameterised by Gx = A^T, Gu = B^T, gamma = f
      // (parallel-solver.hxx:136-147).  It is the ordinary stage step below started from a zero
      // value function (V' = 0, vx' = 0, Vxt' = Vtt' = 0, vt' = 0) -- adding exact zeros.
      for (int i = tid; i < nx; i += T)
        vxn[i] = 0.0;
      for (int e = tid; e < nx * nth; e += T)
        vxt2[e] = 0.0;
      for (int e = tid; e < nth * nth; e += T)
        vtt2[e] = 0.0;
      for (int e = tid; e < nth; e += T)
        vtv2[e] = 0.0;
      ctx.sync();
    } else
    // ---------------- terminal knot (nu = 0): riccati-kernel.hxx:146-149,175-183
    {
      const int trec = nx * nx + nx + nct * nx + nct;
      const int trec_th = trec + nx * d.rec_nth + nct * d.rec_nth + d.rec_nth * d.rec_nth + d.rec_nth; // + [Gx | Gv | Gth | gamma]
      const double *tr = p.term + (size_t)inst * trec_th;
      const double *Qt = tr, *qt = tr + nx * nx, *Ct = qt + nx, *dt = Ct + (size_t)nct * nx;
      double *VN = Vxx_b + (size_t)N * nx * nx;
      for (int m = tid; m < nct * nx; m += T) { // Z = C / mu (stored row-major nct x nx)
        const int r = m / nx, j = m % nx;
        p.fbT[(size_t)inst * nct * nx + m] = Ct[r + (size_t)j * nct] / mu(p, inst);
      }
      for (int m = tid; m < nct; m += T)
        p.ffT[(size_t)inst * nct + m] = dt[m] / mu(p, inst);
      for (int e = tid; e < nx * nx; e += T) { // Vxx = Q + C^T Z
        const int i = e % nx, j = e / nx;
        double acc = 0.0;
        for (int m = 0; m < nct; ++m)
          acc += Ct[m + (size_t)i * nct] * (Ct[m + (size_t)j * nct] / mu(p, inst));
        const double s = Qt[i + j * nx] + acc;
        VN[i + j * nx] = s;
        if (i >= j) {
          Vn[i * d.vs + j] = s;
          Vn[j * d.vs + i] = s;
        }
      }
      for (int i = tid; i < nx; i += T) { // vx = q + C^T z
        double acc = 0.0;
        for (int m = 0; m < nct; ++m)
          acc += Ct[m + (size_t)i * nct] * (dt[m] / mu(p, inst));
        const double s = qt[i] + acc;
        vx_b[(size_t)N * nx + i] = s;
        vxn[i] = s;
      }
      ctx.sync();
      if (N > t_lo) // symmetrised by the step N-1 of the reference (A1); a leg head is not
        for (int e = tid; e < nx * nx; e += T)
          VN[(e % nx) + (e / nx) * nx] = Vn[(e / nx) * d.vs + (e % nx)];
      if (nth > 0) { // nu = 0: Vxt = Gx, Vtt = Gth, vt = gamma (:185-192); Zth = 0 (:146-149)
        const double *Gx = tr + trec, *Gth = Gx + nx * nth + nct * nth, *gam = Gth + nth * nth;
        for (int e = tid; e < nx * nth; e += T) {
          vxt2[e] = Gx[e];
          Vxt_b[(size_t)N * nx * nth + e] = Gx[e];
        }
        for (int e = tid; e < nth * nth; e += T) {
          vtt2[e] = Gth[e];
          Vtt_b[(size_t)N * nth * nth + e] = Gth[e];
        }
        for (int e = tid; e < nth; e += T) {
          vtv2[e] = gam[e];
          vt_b[(size_t)N * nth + e] = gam[e];
        }
        ctx.sync();
      }
    }

    // ---------------- stage knots N-1 .. 0: riccati-kernel.hxx:210-277
    const int nchunk = (d.nt + BLK_CH - 1) / BLK_CH;
    const int nchunk2 = (d.nt2 + BLK_CH - 1) / BLK_CH;
    for (int t = t_first; t >= t_lo; --t) {
      const bool legl = !last_leg && t == t_hi - 1; // the last knot of a parametric leg
      const int gmode = !legmode ? 0 : (legl ? 2 : 1); // parametric blocks: record / zero / leg-last
      double *fbt = fb_b + (size_t)t * nr * nx;
      double *fft = ff_b + (size_t)t * nr;
      // parametric blocks of this knot: from the record (gmode 0), zero (inner knot of a leg),
      // or Gx = A^T, Gu = B^T, Gth = 0, gamma = f (a leg's last knot, parallel-solver.hxx:136-147)
      const double *Am = rec, *Bm = rec + d.off_b;
      const double *Gxr = rec + d.off_gx, *Gur = rec + d.off_gu, *Gvr = rec + d.off_gv, *Gthr = rec + d.off_gth,
                   *gamr = rec + d.off_gam, *fr = rec + d.off_f;
      auto gx = [&](int i, int j) { return gmode == 0 ? Gxr[i + j * nx] : (gmode == 2 ? Am[j + i * nx] : 0.0); };
      auto gu = [&](int c, int j) { return gmode == 0 ? Gur[c + j * nu] : (gmode == 2 ? Bm[j + c * nx] : 0.0); };
      auto gv = [&](int m, int j) { return gmode == 0 ? Gvr[m + j * nc] : 0.0; };
      auto gth = [&](int e) { return gmode == 0 ? Gthr[e] : 0.0; };
      auto gam = [&](int i) { return gmode == 0 ? gamr[i] : (gmode == 2 ? fr[i] : 0.0); };
      const double *Vxtn = vxt2 + thcur * nx * nth, *Vttn = vtt2 + thcur * nth * nth, *vtn = vtv2 + thcur * nth;
      const int thc = nx + 1; // first theta column of X / KK
      AB2_CLK(9);
      ctx.wait_copy(0);
      AB2_CLK(0);
      // (1) W = V' M (+ vx' on the affine column), :216-224, computed as W^T = M^T V' (V' symmetric):
      // the operand with the awkward shared-memory stride -- a column of M, nx doubles apart in the
      // record, 2-way bank conflicts for odd and for 8-aligned nx alike -- is then the A operand,
      // loaded ONCE per k-step, and the four B operands are rows of V' (stride 4 or 12 mod 16:
      // conflict-free).  Work item = (n-tile of M's columns, chunk of four m-tiles of state rows).
      // No predicates inside: padding columns of M point at the zeroed slack, padding rows of the
      // contraction meet the zero columns of V'.
      const int nchunk_m = (d.mtx + BLK_CH - 1) / BLK_CH;
      for (int it = warp; it < d.nt * nchunk_m; it += NW) {
        const int nt = it / nchunk_m, m0 = (it % nchunk_m) * BLK_CH;
        const int nrow = d.mtx - m0; // warp-uniform
        double acc[BLK_CH][2];
        const double *vp[BLK_CH];
        AB2_UNROLL
        for (int c = 0; c < BLK_CH; ++c) {
          acc[c][0] = acc[c][1] = 0.0;
          vp[c] = Vn + (8 * (m0 + (c < nrow ? c : 0)) + g) * d.vs + q;
        }
        const double *mp = rec + blk_col_offset(d, 8 * nt + g) + q;
        if (nrow >= BLK_CH) {
          for (int kt = 0; kt < d.kt; ++kt) {
            const double ma = mp[4 * kt];
            AB2_UNROLL
            for (int c = 0; c < BLK_CH; ++c)
              ctx.mma(acc[c], ma, vp[c][4 * kt]);
          }
        } else {
          for (int kt = 0; kt < d.kt; ++kt) {
            const double ma = mp[4 * kt];
            AB2_UNROLL
            for (int c = 0; c < BLK_CH; ++c)
              if (c < nrow)
                ctx.mma(acc[c], ma, vp[c][4 * kt]);
          }
        }
        const int jp = 8 * nt + g; // logical column of W held by this lane
        AB2_UNROLL
        for (int c = 0; c < BLK_CH; ++c)
          if (c < nrow) {
            AB2_UNROLL
            for (int e = 0; e < 2; ++e) {
              const int i = 8 * (m0 + c) + 2 * q + e;
              if (i < nx)
                Wsm[i * d.sw + jp] = acc[c][e] + (jp == nx ? vxn[i] : 0.0);
            }
          }
      }
      ctx.sync();
      AB2_CLK(1);
      if (two_parts)
        ctx.wait_copy(1);
      // (2) H = H0 + M^T W  -> Hs, :226-241
      for (int it = warp; it < d.nt * nchunk; it += NW) {
        const int mt = it / nchunk, n0 = (it % nchunk) * BLK_CH;
        const int ncol = d.nt - n0;
        double acc[BLK_CH][2];
        AB2_UNROLL
        for (int c = 0; c < BLK_CH; ++c) {
          AB2_UNROLL
          for (int e = 0; e < 2; ++e) {
            const int o = (c < ncol) ? blk_h0_offset(d, 8 * mt + g, 8 * (n0 + c) + 2 * q + e) : -1;
            const double hv = rec[o >= 0 ? o : 0];
            acc[c][e] = (o >= 0) ? hv : 0.0;
          }
        }
        const double *ap = rec + blk_col_offset(d, 8 * mt + g) + q; // M^T: row = column of M
        const double *wp = Wsm + q * d.sw + 8 * n0 + g;
        if (ncol >= BLK_CH) {
          for (int kt = 0; kt < d.kt; ++kt) {
            const double mv = ap[4 * kt];
            const double ma = (4 * kt + q < nx) ? mv : 0.0; // W's rows beyond nx are not W
            AB2_UNROLL
            for (int c = 0; c < BLK_CH; ++c)
              ctx.mma(acc[c], ma, wp[4 * kt * d.sw + 8 * c]);
          }
        } else {
          for (int kt = 0; kt < d.kt; ++kt) {
            const double mv = ap[4 * kt];
            const double ma = (4 * kt + q < nx) ? mv : 0.0;
            AB2_UNROLL
            for (int c = 0; c < BLK_CH; ++c)
              if (c < ncol)
                ctx.mma(acc[c], ma, wp[4 * kt * d.sw + 8 * c]);
          }
        }
        AB2_UNROLL
        for (int c = 0; c < BLK_CH; ++c)
          if (c < ncol)
            sts2(Hs + (8 * mt + g) * d.sh + 8 * (n0 + c) + 2 * q, acc[c][0], acc[c][1]);
      }
      ctx.sync();
      AB2_CLK(2);
      // (3) X = [Shat^T rhat; C d] (nk rows, columns 0..nx) and the KKT matrix, :232-257
      for (int e = tid; e < nk * (nx + 1); e += T) {
        const int c = e / (nx + 1), j = e % (nx + 1);
        double v;
        if (c < nu)
          v = Hs[(nx + 1 + c) * d.sh + j];
        else
          v = (j < nx) ? rec[d.off_c + j * nc + (c - nu)] : rec[d.off_dv + (c - nu)];
        X[c * d.sx + j] = v;
      }
      for (int e = tid; e < nk * nk; e += T) {
        const int r = e % nk, c = e / nk;
        double v = 0.0;
        if (r < nu && c < nu)
          v = Hs[(nx + 1 + r) * d.sh + (nx + 1 + c)];
        else if (r >= nu && c < nu)
          v = rec[d.off_d + c * nc + (r - nu)];
        else if (r >= nu && c >= nu)
          v = (r == c) ? -mu(p, inst) : 0.0;
        kkt[r + c * nk] = v;
      }
      if (nth > 0) {
        // (8a) parametric right-hand sides, riccati-kernel.hxx:284-291: Gxhat = Gx + A^T Vxt',
        // Guhat = Gu + B^T Vxt'; [Guhat; Gv] become the columns nx+1.. of X, so the solves below produce
        // [Kth; Zth] together with [K k; Z z] (same factor, same routine, all the CTA's warps)
        const int nxu = nx + nu;
        for (int e = tid; e < nxu * nth; e += T) {
          const int j = e / nxu, r = e - j * nxu;
          const bool isx = r < nx;
          const int i = isx ? r : r - nx;
          const double *Mc = isx ? Am + i * nx : Bm + i * nx; // column i of A / B
          const double *vc = Vxtn + j * nx;
          double a0 = 0.0, a1 = 0.0;
          int c = 0;
          for (; c + 2 <= nx; c += 2) {
            a0 += Mc[c] * vc[c];
            a1 += Mc[c + 1] * vc[c + 1];
          }
          if (c < nx)
            a0 += Mc[c] * vc[c];
          const double acc = a0 + a1;
          if (isx)
            gxh[i + j * nx] = gx(i, j) + acc;
          else
            X[i * d.sx + thc + j] = gu(i, j) + acc;
        }
        for (int e = tid; e < nc * nth; e += T) {
          const int m = e / nth, j = e - m * nth;
          X[(nu + m) * d.sx + thc + j] = gv(m, j);
        }
      }
      ctx.sync();
      // the tail of the record (cost blocks, C, D, d) is consumed: fetch the next knot's
      if (two_parts && t > t_lo) {
        const double *src = stage_b + (size_t)stage_slot(p, t - 1) * d.srec_pad;
        ctx.issue_copy(1, rec + d.split, src + d.split, d.srec_pad - d.split);
      }
      // Unconstrained knots (SPD Rhat): the branch-free warp LDL^T; anything that needs an
      // interchange or a 2x2 pivot falls back to the general cooperative algorithm on a copy.
      AB2_CLK(3);
      // unconstrained knots: LDL^T by the whole CTA (vote per column), else the general algorithm on a copy
      const bool cta_fast = nc == 0 && nk <= 32 && nk * nk <= d.xrows * d.sx;
      const bool try_fast = !cta_fast && nc == 0 && nk <= 32 && nk * nk <= d.xrows * d.sx;
      constexpr int SNK = D::static_nk;
      const bool regs_pad = SNK == 0 && cta_fast && nk <= 16; // register path, identity-padded to 8 / 16
      const bool need_copy = try_fast || (cta_fast && SNK == 0 && !regs_pad);
      if (need_copy)
        for (int e = tid; e < nk * nk; e += T)
          Ys[e] = kkt[e]; // Y is free until the solves
      if (need_copy)
        ctx.sync();
      int fast_regs = 0; // the pivot-free LDL^T succeeded (uniform over the CTA)
      if constexpr (SNK > 0) { // compile-time size: one warp, rows in registers; the others wait at the barrier
        if (warp == 0)
          fast_regs = ldlt_regs_warp<SNK>(ctx, kkt, dd, sd, perm, kind) ? 1 : 0;
        fast_regs = ctx.sync_or(fast_regs); // (the matrix is untouched on failure)
      } else if (regs_pad) {
        if (warp == 0)
          fast_regs = (nk <= 8 ? ldlt_regs_warp_pad<8>(ctx, kkt, nk, dd, sd, perm, kind)
                               : ldlt_regs_warp_pad<16>(ctx, kkt, nk, dd, sd, perm, kind))
                          ? 1
                          : 0;
        fast_regs = ctx.sync_or(fast_regs); // (the matrix is untouched on failure)
      } else if (cta_fast) {
        fast_regs = ldlt_fast_cta(ctx, kkt, nk, dd, sd, perm, kind) ? 1 : 0;
        if (!fast_regs) {
          for (int e = tid; e < nk * nk; e += T)
            kkt[e] = Ys[e];
          ctx.sync();
        }
      }
      const bool need_general = !fast_regs;
      if (need_general && tid < bk_threads) { // the other warps go straight to the CTA barrier below
        bool done = false;
        if (try_fast) { // (bk_threads == 32: warp 0)
          done = ldlt_fast_warp(ctx, kkt, nk, dd, sd, perm, kind);
          if (!done)
            for (int e = lane; e < nk * nk; e += 32)
              kkt[e] = Ys[e];
        }
        if (!done && !bk_factor_group<16>(grp, kkt, nk, nk, dd, sd, perm, kind, pv))
          st |= ST_STAGE_FACTOR_FAILED;
      }
      ctx.sync();
      AB2_CLK(4);
      // column tid of [K k; Z z] = -KKT^-1 X[:, tid]
      // (four lanes per column with butterfly reductions would issue more instructions without
      // shortening the chains, which are latency-bound)
      if (fast_regs && nk <= 32) // identity interchanges, 1x1 pivots: every warp solves a chunk of columns
        ldlt_solve_rows_warp(ctx, kkt, nk, dd, X, KKs, d.sx, nx + 1 + nth);
      else
        for (int col = tid; col < nx + 1 + nth; col += T)
          bk_solve_column_rt(kkt, nk, dd, sd, perm, kind, X + col, Ys + col, KKs + col, d.sx);
      ctx.sync();
      AB2_CLK(5);
      for (int e = tid; e < nk * nx; e += T) // gains K, Z (row-major nk x nx)
        fbt[e] = KKs[(e / nx) * d.sx + (e % nx)];
      for (int c = tid; c < nk; c += T)
        fft[c] = KKs[c * d.sx + nx];
      // (4) [Ahat a] = [A f] + B KK (:266-267) and (5) [Vxx vx] = [Qhat qhat] + X^T KK (:270-277)
      for (int it = warp; it < d.mtx * nchunk2; it += NW) {
        const int mt = it / nchunk2, n0 = (it % nchunk2) * BLK_CH;
        const int i = 8 * mt + g, ic = i < nx ? i : 0;
        double EA[BLK_CH][2], VV[BLK_CH][2];
        AB2_UNROLL
        for (int c = 0; c < BLK_CH; ++c) {
          AB2_UNROLL
          for (int e = 0; e < 2; ++e) {
            const int jj = 8 * (n0 + c) + 2 * q + e;
            const bool in = (n0 + c < d.nt2) && i < nx && jj <= nx;
            const int jc = in ? jj : 0;
            const double ev = rec[blk_col_offset(d, jc) + ic];
            const double hv = Hs[ic * d.sh + jc];
            EA[c][e] = in ? ev : 0.0;
            VV[c][e] = in ? hv : 0.0;
          }
        }
        // KK rows >= nk meet zero operands, KK columns > nx feed outputs nobody stores:
        // no predicate on the KK fragments
        const double *bp = rec + d.off_b + ic;
        const double *xp = X + ic;
        const double *kp = KKs + q * d.sx + 8 * n0 + g;
        const int ncol = d.nt2 - n0;
        for (int k2 = 0; k2 < d.kt2; ++k2) {
          const int c4 = 4 * k2 + q;
          const double bv = bp[(c4 < nu ? c4 : 0) * nx];
          const double bf = (c4 < nu && i < nx) ? bv : 0.0;
          const double xr = xp[c4 * d.sx];
          const double xf = (c4 < nk && i < nx) ? xr : 0.0;
          AB2_UNROLL
          for (int c = 0; c < BLK_CH; ++c)
            if (c < ncol) {
              const double kf = kp[4 * k2 * d.sx + 8 * c];
              ctx.mma(EA[c], bf, kf);
              ctx.mma(VV[c], xf, kf);
            }
        }
        if (i < nx) {
          AB2_UNROLL
          for (int c = 0; c < BLK_CH; ++c)
            if (n0 + c < d.nt2) {
              AB2_UNROLL
              for (int e = 0; e < 2; ++e) {
                const int jj = 8 * (n0 + c) + 2 * q + e;
                if (jj < nx) {
                  // (the third block of a leg's terminal knot is never written by the reference, A6)
                  fbt[(nk + i) * nx + jj] = legl ? 0.0 : EA[c][e];
                  if (t == t_lo) // datas[0].Vxx -- and every leg head -- is left unsymmetrised (A1)
                    Vxx_b[(size_t)t * nx * nx + i + jj * nx] = VV[c][e];
                  if (i >= jj) { // V' = lower triangle mirrored (:216 of the next step)
                    Vn[i * d.vs + jj] = VV[c][e];
                    Vn[jj * d.vs + i] = VV[c][e];
                  }
                } else if (jj == nx) {
                  fft[nk + i] = legl ? 0.0 : EA[c][e];
                  vx_b[(size_t)t * nx + i] = VV[c][e];
                  vxn[i] = VV[c][e];
                }
              }
            }
        }
      }
      ctx.sync();
      AB2_CLK(6);
      if (nth > 0) {
        // (8b) parametric value function, riccati-kernel.hxx:293-311.  With Ahat = A + B K and
        // a = f + B k the reference's sums regroup exactly into the forms it keeps in comments (:297, :301):
        //   vt  = (gamma + vt') + Guhat^T k + Vxt'^T f,   Vxt = Gxhat + K^T Guhat,
        //   Vtt = (Gth + Vtt') + Guhat^T Kth
        // (Guhat sits in X's theta columns, [Kth; Zth] in KK's): four independent loops, one barrier.
        double *Vxtc = vxt2 + (thcur ^ 1) * nx * nth, *Vttc = vtt2 + (thcur ^ 1) * nth * nth,
               *vtc = vtv2 + (thcur ^ 1) * nth;
        double *ftt = fth_b + (size_t)t * nr * nth;
        const double *Gh = X + thc, *Kt = KKs + thc; // Guhat[c][j] = Gh[c*sx + j], Kth[c][j] = Kt[c*sx + j]
        for (int e = tid; e < nk * nth; e += T) { // fth rows [Kth; Zth]
          const int r = e / nth, j = e - r * nth;
          ftt[e] = Kt[r * d.sx + j];
        }
        for (int e = tid; e < nx * nth; e += T) { // Yth = B Kth
          const int i = e / nth, j = e - i * nth;
          double acc = 0.0;
          for (int c = 0; c < nu; ++c)
            acc += Bm[i + c * nx] * Kt[c * d.sx + j];
          ftt[nk * nth + e] = legl ? 0.0 : acc; // (never written on a leg's terminal knot)
        }
        for (int i = tid; i < nth; i += T) {
          const double s0 = gam(i) + vtn[i];
          double s1 = 0.0, s2 = 0.0;
          for (int c = 0; c < nu; ++c)
            s1 += Gh[c * d.sx + i] * KKs[c * d.sx + nx];
          for (int c = 0; c < nx; ++c)
            s2 += Vxtn[c + i * nx] * fr[c];
          const double v = (s0 + s1) + s2;
          vtc[i] = v;
          vt_b[(size_t)t * nth + i] = v;
        }
        for (int e = tid; e < nx * nth; e += T) {
          const int j = e / nx, i = e - j * nx;
          double s1 = 0.0;
          for (int c = 0; c < nu; ++c)
            s1 += KKs[c * d.sx + i] * Gh[c * d.sx + j];
          const double v = gxh[e] + s1;
          Vxtc[e] = v;
          Vxt_b[(size_t)t * nx * nth + e] = v;
        }
        for (int e = tid; e < nth * nth; e += T) {
          const int j = e / nth, i = e - j * nth;
          double s1 = 0.0;
          for (int c = 0; c < nu; ++c)
            s1 += Gh[c * d.sx + i] * Kt[c * d.sx + j];
          const double v = (gth(e) + Vttn[e]) + s1;
          Vttc[e] = v;
          Vtt_b[(size_t)t * nth * nth + e] = v;
        }
        thcur ^= 1;
        ctx.sync();
      }
      AB2_CLK(7);
      if (t > t_lo) {
        const double *src = stage_b + (size_t)stage_slot(p, t - 1) * d.srec_pad;
        ctx.issue_copy(0, rec, src, d.split);
        double *Vt = Vxx_b + (size_t)t * nx * nx; // symmetric Vxx_t, as the next step leaves it
        for (int e = tid; e < nx * nx; e += T)
          Vt[e] = Vn[(e / nx) * d.vs + (e % nx)];
      }
    }

    // ---------------- initial stage: proximal-riccati.hxx:42-55 (nth = 0)
    // (leg mode: the condensed block-tridiagonal system takes its place, condensed_solve below)
    if (!legmode) {
      const int n0 = nx + nc0;
      double *K0 = sm; // n0 x n0 column-major (overlays the stage buffers)
      double *b0 = K0 + n0 * n0;
      double *x0w = b0 + n0;
      double *dd0 = x0w + n0;
      double *sd0 = dd0 + n0;
      double *o0 = sd0 + n0;
      int *perm0 = reinterpret_cast<int *>(o0 + n0);
      int *kind0 = perm0 + n0;
      ctx.sync(); // Vxx_0 / vx_0 of this instance are in global memory, written by this CTA
      const double *G0 = p.G0 + (size_t)inst * nc0 * nx;
      const double *g0 = p.g0 + (size_t)inst * nc0;
      for (int e = tid; e < n0 * n0; e += T) {
        const int i = e % n0, j = e / n0;
        double v = 0.0;
        if (i >= j) {
          if (i < nx)
            v = Vxx_b[i + j * nx]; // lower triangle of Vxx_0
          else if (j < nx)
            v = G0[(i - nx) + (size_t)j * nc0];
        }
        K0[e] = v;
      }
      for (int i = tid; i < n0; i += T)
        b0[i] = (i < nx) ? -vx_b[i] : -g0[i - nx];
      ctx.sync();
      CtaAsGroup<Ctx> grp0{ctx, tid, 32 * ((n0 + 31) / 32)};
      if (tid < grp0.nthreads) {
        if (!bk_factor_group<8>(grp0, K0, n0, n0, dd0, sd0, perm0, kind0, pv))
          st |= ST_INIT_FACTOR_FAILED;
        bk_solve_vec_group(grp0, K0, n0, n0, dd0, sd0, perm0, kind0, b0, x0w, o0);
      }
      ctx.sync();
      for (int i = tid; i < n0; i += T)
        p.kkt0[(size_t)inst * n0 + i] = o0[i];
      ctx.sync();
      if (nth > 0) { // fth = -K0^-1 [Vxt_0; 0], thGrad, thHess (proximal-riccati.hxx:50-59)
        const double *Vxt0 = vxt2 + thcur * nx * nth, *Vtt0 = vtt2 + thcur * nth * nth, *vt0 = vtv2 + thcur * nth;
        for (int e = tid; e < n0 * nth; e += T) {
          const int r = e / nth, j = e % nth;
          trhs[e] = (r < nx) ? Vxt0[r + j * nx] : 0.0;
        }
        ctx.sync();
        if (tid < nth)
          bk_solve_column_rt(K0, n0, dd0, sd0, perm0, kind0, trhs + tid, twork + tid, tsol + tid, nth);
        ctx.sync();
        for (int e = tid; e < n0 * nth; e += T)
          p.kkt0fth[(size_t)inst * n0 * nth + e] = tsol[e];
        for (int i = tid; i < nth; i += T) {
          double acc = 0.0;
          for (int c = 0; c < nx; ++c)
            acc += Vxt0[c + i * nx] * o0[c];
          p.thGrad[(size_t)inst * nth + i] = vt0[i] + acc;
        }
        for (int e = tid; e < nth * nth; e += T) {
          const int i = e % nth, j = e / nth;
          double acc = 0.0;
          for (int c = 0; c < nx; ++c)
            acc += Vxt0[c + i * nx] * tsol[c * nth + j];
          p.thHess[(size_t)inst * nth * nth + e] = Vtt0[e] + acc;
        }
        ctx.sync();
      }
    }
    if (tid == 0) {
      if (legmode) { // several CTAs report on one instance (the host clears both words first)
        ctx.atomic_or(p.status + inst, st);
        if (p.pivstat)
          ctx.atomic_add(p.pivstat + inst, pv);
      } else {
        p.status[inst] = st;
        if (p.pivstat)
          p.pivstat[inst] = pv;
      }
    }
  }

  // ---------------- forward rollout: riccati-kernel.hxx:196-207, 315-377
  if (p.do_fwd) {
    const int n0 = nx + nc0;
    const double *k0 = p.kkt0 + (size_t)inst * n0;
    double *xs_b = p.xs + (size_t)inst * (N + 1) * nx;
    double *us_b = p.us + (size_t)inst * N * nu;
    double *vs_b = p.vs + (size_t)inst * N * nc;
    double *lb_b = p.lbdas + (size_t)inst * N * nx;
    const int RING = d.fwd_ring, FS = d.fwd_slot;
    const int R = nr * nx;
    double *ring = sm;
    double *xc = sm + RING * FS;
    double *xnx = xc + blk_ev(nx);
    // generic-proxy writes of the backward pass (fb in global memory, the initial-stage
    // workspace in shared memory) ordered before the ring's bulk copies read / overwrite them
    ctx.proxy_fence();
    ctx.sync();
    // fb record of knot t -> ring slot s by one TMA bulk copy.  A record that starts at an
    // odd double (odd-sized records) is fetched from the aligned double before it; the
    // record then sits one double into the slot.
    const size_t e_inst = (size_t)inst * N * R;
    // (parity of the ABSOLUTE address: a batch slice may start at an odd double of the array)
    auto rec_shift = [&](int t) {
      return (int)((reinterpret_cast<uintptr_t>(p.fb + e_inst + (size_t)t * R) >> 3) & 1);
    };
    auto fill_slot = [&](int s_, int t) {
      const int a = rec_shift(t);
      ctx.issue_copy(s_, ring + s_ * FS, p.fb + (e_inst + (size_t)t * R - a), blk_ev(R + a));
    };
    // stage knots of this CTA: [t_lo, t_s1) (all of them outside leg mode); a parametric leg's
    // last knot t_hi - 1 yields u and v only (riccati-kernel.hxx:352-353)
    const int t_s1 = last_leg ? N : t_hi;
    for (int s_ = 0; s_ < RING && t_lo + s_ < t_s1; ++s_)
      fill_slot(s_, t_lo + s_);
    // theta terms of the rollout (riccati-kernel.hxx:196-207, 315-377): only when theta is given.
    // Leg mode: theta = the co-state at the head of the NEXT leg, x and lbda at this leg's head =
    // blocks of the condensed solution (parallel-solver.hxx:214-238).
    const double *condv = legmode ? p.cond + (size_t)inst * (nc0 + nx * (2 * NLEG - 1)) : nullptr;
    const double *theta = legmode ? (last_leg ? nullptr : condv + cond_offset(2 * (leg + 1), nc0, nx))
                                  : ((nth > 0 && p.theta) ? p.theta + (size_t)inst * nth : nullptr);
    const double *f0th = (theta && !legmode) ? p.kkt0fth + (size_t)inst * n0 * nth : nullptr;
    const double *fthf = theta ? p.fth + (size_t)inst * N * nr * nth : nullptr;
    const double *Vxtf = theta ? p.Vxt + (size_t)inst * (N + 1) * nx * nth : nullptr;
    if (legmode) {
      const double *xh = condv + cond_offset(2 * leg + 1, nc0, nx), *lh = condv + cond_offset(2 * leg, nc0, nx);
      for (int i = tid; i < nx; i += T) {
        xc[i] = xh[i];
        xs_b[(size_t)t_lo * nx + i] = xh[i];
        if (leg > 0)
          lb_b[(size_t)(t_lo - 1) * nx + i] = lh[i];
      }
      if (leg == 0)
        for (int m = tid; m < nc0; m += T)
          p.lbd0[(size_t)inst * nc0 + m] = lh[m];
    } else {
    for (int i = tid; i < nx; i += T) {
      double v = k0[i];
      if (theta) {
        double acc = 0.0;
        for (int c = 0; c < nth; ++c)
          acc += f0th[i * nth + c] * theta[c];
        v += acc;
      }
      xc[i] = v;
      xs_b[i] = v;
    }
    for (int m = tid; m < nc0; m += T) {
      double v = k0[nx + m];
      if (theta) {
        double acc = 0.0;
        for (int c = 0; c < nth; ++c)
          acc += f0th[(nx + m) * nth + c] * theta[c];
        v += acc;
      }
      p.lbd0[(size_t)inst * nc0 + m] = v;
    }
    }
    // lbda_t = vx_t + Vxx_t x_t (t >= 1; Vxx_t symmetric: element (c, i) read as (i, c) keeps
    // the loads of neighbouring threads contiguous).  Runs on the warps pass 1 leaves idle.
    const int lam0 = 32 * ((nr + 31) / 32);
    const bool lam_overlap = T - lam0 >= 32;
    auto lam_rows = [&](int tt, const double *x, int first, int step) {
      const double *V = Vxx_b + (size_t)tt * nx * nx;
      for (int i = first; i < nx; i += step) {
        double s0 = vx_b[(size_t)tt * nx + i], s1 = 0.0;
        int c = 0;
        for (; c + 1 < nx; c += 2) {
          s0 += V[(size_t)c * nx + i] * x[c];
          s1 += V[(size_t)(c + 1) * nx + i] * x[c + 1];
        }
        if (c < nx)
          s0 += V[(size_t)c * nx + i] * x[c];
        double lam = s0 + s1;
        if (theta) {
          double acc = 0.0;
          for (int c2 = 0; c2 < nth; ++c2)
            acc += Vxtf[(size_t)tt * nx * nth + i + c2 * nx] * theta[c2];
          lam += acc;
        }
        lb_b[(size_t)(tt - 1) * nx + i] = lam;
      }
    };
    // Pass 1: x_{t+1} = a + Ahat x_t (and u, v): thread r owns gain row r (nr <= T).
    double gff = (tid < nr && t_lo < t_s1) ? ff_b[(size_t)t_lo * nr + tid] : 0.0;
    ctx.sync();
    for (int t = t_lo; t < t_s1; ++t) {
      const int s_ = (t - t_lo) % RING;
      const bool legl = !last_leg && t == t_hi - 1;
      ctx.wait_copy(s_);
      const double *slot = ring + s_ * FS + rec_shift(t);
      if (tid < nr) {
        const int r = tid;
        double s0 = gff, s1 = 0.0;
        int c = 0;
        for (; c + 1 < nx; c += 2) {
          s0 += slot[r * nx + c] * xc[c];
          s1 += slot[r * nx + c + 1] * xc[c + 1];
        }
        if (c < nx)
          s0 += slot[r * nx + c] * xc[c];
        double sv = s0 + s1;
        if (theta) {
          double acc = 0.0;
          for (int c2 = 0; c2 < nth; ++c2)
            acc += fthf[((size_t)t * nr + r) * nth + c2] * theta[c2];
          sv += acc;
        }
        if (r < nu)
          us_b[(size_t)t * nu + r] = sv;
        else if (r < nk)
          vs_b[(size_t)t * nc + (r - nu)] = sv;
        else if (!legl) { // (the state at the next leg's head comes from the condensed solution)
          xnx[r - nk] = sv;
          xs_b[(size_t)(t + 1) * nx + (r - nk)] = sv;
        }
        gff = (t + 1 < t_s1) ? ff_b[(size_t)(t + 1) * nr + r] : 0.0;
      } else if (lam_overlap && tid >= lam0 && t > t_lo) {
        lam_rows(t, xc, tid - lam0, T - lam0);
      }
      double *tmp = xc;
      xc = xnx;
      xnx = tmp;
      ctx.sync(); // x_{t+1} visible; everyone is done with x_t and with this slot
      if (t + RING < t_s1)
        fill_slot(s_, t + RING);
    }
    if (lam_overlap) {
      if (last_leg && N > t_lo)
        lam_rows(N, xc, tid, T);
    } else {
      for (int tt = t_lo + 1; tt <= (last_leg ? N : t_hi - 1); ++tt) // xs is in global memory, written by this CTA
        lam_rows(tt, xs_b + (size_t)tt * nx, tid, T);
    }
    if (last_leg)
    // terminal multipliers v_N = z + Z x_N
    for (int m = tid; m < nct; m += T) {
      double s = p.ffT[(size_t)inst * nct + m];
      for (int c = 0; c < nx; ++c)
        s += p.fbT[(size_t)inst * nct * nx + (size_t)m * nx + c] * xc[c];
      p.vsT[(size_t)inst * nct + m] = s;
    }
    ctx.sync();
  }
}

// ---------------------------------------------------------------------------
// Leg mode, step 2: the condensed system of one instance (the "boundary consensus" of the
// legs).  Restates ParallelRiccatiSolver::assembleCondensedSystem + the solve + the iterative
// refinement of ::backward (gar/parallel-solver.hxx:85-129, 166-203) on top of
// symmetricBlockTridiagSolve / blockTridiagMatMul / blockTridiagRefinementStep
// (gar/block-tridiagonal.hpp:82-138, 52-75, 147-182), one CTA per instance, everything in
// shared memory.  Unknowns [lbda_0 | x_0 | theta_0 | x_{h1} | theta_1 | x_{h2} | ...]
// (h_j = head knot of leg j, theta_{j-1} = lbda_{h_j}); block b = 2j+1 is x_{h_j}, b = 2j
// (j >= 1) is theta_{j-1}:
//   diagonal   D_0 = 0,  D_{2j+1} = Vxx[h_j] (as stored, lower triangle factored),  D_{2j} = Vtt[h_{j-1}]
//   super      S_0 = G0, S_{2j+1} = Vxt[h_j],                                        S_{2j} = -I
//   rhs        -g0,      -vx[h_j],                                                   -vt[h_{j-1}]
// Backward-looking block U D U^T with one Bunch-Kaufman per diagonal block, then at most
// `max_refine` refinement steps until the residual's infinity norm is <= thr.
// (The reference's first refinement pass starts from a stale error buffer -- condensedErr is
// only reset at the END of a pass, :201 -- which on a fresh solver zeroes the solution and
// re-solves it; the intended algorithm is what runs here: identical to rounding.)
// Writes p.cond (the solution), p.kkt0 = [x_0; lbda_0]; a failed block factorisation sets
// ST_CONDENSED_FACTOR_FAILED and leaves the solve where the reference's early return does.
AB2_HD constexpr int condensed_smem_doubles(int nx, int nc0, int T) {
  const int NB = 2 * T, dmax = nx > nc0 ? nx : nc0, TD = nc0 + nx * (2 * T - 1);
  return NB * dmax * dmax + (NB - 1) * dmax * dmax + NB * (3 * dmax + 2) + 2 * blk_ev(TD) + dmax * dmax + 2 * blk_ev(dmax);
}

template <class Ctx>
AB2_D void condensed_solve(Ctx &ctx, const SweepParams &p, const int nx, const int inst, double *__restrict__ sm,
                           const int max_refine = 5, const double thr = 1e-10) {
  const int tid = ctx.tid, NT_ = ctx.nthreads;
  const int N = p.N, nc0 = p.nc0, T = p.legs, nth = nx;
  const int NB = 2 * T, dmax = nx > nc0 ? nx : nc0, TD = nc0 + nx * (2 * T - 1);
  const int blk = dmax * dmax, auxs = 3 * dmax + 2;
  double *Df = sm;
  double *U = Df + (size_t)NB * blk;
  double *aux = U + (size_t)(NB - 1) * blk;
  double *sol = aux + (size_t)NB * auxs;
  double *err = sol + blk_ev(TD);
  double *wk = err + blk_ev(TD);
  double *vw = wk + blk; // 2 * ev(dmax): work + out of the vector solves
  auto dm = [&](int b) { return b == 0 ? nc0 : nx; };
  auto off = [&](int b) { return cond_offset(b, nc0, nx); };
  auto head = [&](int j) { return leg_begin(N, j, T); };
  const double *Vxx_b = p.Vxx + (size_t)inst * (N + 1) * nx * nx;
  const double *vx_b = p.vx + (size_t)inst * (N + 1) * nx;
  const double *Vxt_b = p.Vxt + (size_t)inst * (N + 1) * nx * nth;
  const double *Vtt_b = p.Vtt + (size_t)inst * (N + 1) * nth * nth;
  const double *vt_b = p.vt + (size_t)inst * (N + 1) * nth;
  const double *G0 = p.G0 + (size_t)inst * nc0 * nx;
  const double *g0 = p.g0 + (size_t)inst * nc0;
  // original blocks (global memory)
  auto Dorig = [&](int b) -> const double * { // nullptr = zero block
    if (b == 0)
      return nullptr;
    return (b & 1) ? Vxx_b + (size_t)head(b / 2) * nx * nx : Vtt_b + (size_t)head(b / 2 - 1) * nth * nth;
  };
  auto Sup = [&](int b) -> const double * { // nullptr = -I (even b >= 2)
    if (b == 0)
      return G0;
    return (b & 1) ? Vxt_b + (size_t)head(b / 2) * nx * nth : nullptr;
  };
  auto rhs_at = [&](int b, int i) {
    if (b == 0)
      return -g0[i];
    return (b & 1) ? -vx_b[(size_t)head(b / 2) * nx + i] : -vt_b[(size_t)head(b / 2 - 1) * nth + i];
  };
  // y (dm(b)) -= S_b x (dm(b+1))
  auto sub_Sx = [&](int b, double *y, const double *x) {
    const double *S = Sup(b);
    const int r = dm(b), c = dm(b + 1);
    for (int i = tid; i < r; i += NT_) {
      double acc = 0.0;
      if (S) {
        for (int k = 0; k < c; ++k)
          acc += S[i + (size_t)k * r] * x[k];
      } else {
        acc = -x[i];
      }
      y[i] -= acc;
    }
  };
  CtaAsGroup<Ctx> grp{ctx, tid, NT_};
  int st = 0, pv = 0;
  auto bptr = [&](int b) { return Df + (size_t)b * blk; };
  auto uptr = [&](int b) { return U + (size_t)b * blk; };
  auto dd_ = [&](int b) { return aux + (size_t)b * auxs; };
  auto sd_ = [&](int b) { return aux + (size_t)b * auxs + dmax; };
  auto pm_ = [&](int b) { return reinterpret_cast<int *>(aux + (size_t)b * auxs + 2 * dmax); };
  auto kd_ = [&](int b) { return reinterpret_cast<int *>(aux + (size_t)b * auxs + 2 * dmax) + dmax; };
  // x (dm(b)) = D_b^-1 x  with the factor of block b
  auto solve_vec = [&](int b, double *x) {
    const int n = dm(b);
    if (n == 0)
      return;
    bk_solve_vec_group(grp, bptr(b), n, n, dd_(b), sd_(b), pm_(b), kd_(b), x, vw, vw + blk_ev(dmax));
    for (int i = tid; i < n; i += NT_)
      x[i] = vw[blk_ev(dmax) + i];
    ctx.sync();
  };
  // ---- assemble
  for (int b = 0; b < NB; ++b) {
    const double *Do = Dorig(b);
    const int n = dm(b);
    for (int e = tid; e < n * n; e += NT_)
      bptr(b)[e] = Do ? Do[e] : 0.0;
    for (int i = tid; i < n; i += NT_)
      sol[off(b) + i] = rhs_at(b, i);
    if (b + 1 < NB) { // U_b = S_b^T: dm(b+1) x dm(b)
      const double *S = Sup(b);
      const int r = dm(b + 1), c = n;
      for (int e = tid; e < r * c; e += NT_) {
        const int i = e % r, j = e / r; // U(i, j) = S(j, i)
        uptr(b)[e] = S ? S[j + (size_t)i * c] : (i == j ? -1.0 : 0.0);
      }
    }
  }
  ctx.sync();
  // ---- symmetricBlockTridiagSolve (block-tridiagonal.hpp:99-135)
  bool ok = true;
  for (int i = NB - 2; i >= 0 && ok; --i) {
    const int n1 = dm(i + 1), n0 = dm(i);
    if (!bk_factor_group<8>(grp, bptr(i + 1), n1, n1, dd_(i + 1), sd_(i + 1), pm_(i + 1), kd_(i + 1), pv)) {
      ok = false;
      break;
    }
    solve_vec(i + 1, sol + off(i + 1));
    sub_Sx(i, sol + off(i), sol + off(i + 1));
    // U_i = D_{i+1}^-1 U_i, column by column (thread j owns column j)
    for (int j0 = 0; j0 < n0; j0 += NT_) {
      const int j = j0 + tid;
      if (j < n0)
        bk_solve_column_rt(bptr(i + 1), n1, dd_(i + 1), sd_(i + 1), pm_(i + 1), kd_(i + 1), uptr(i) + (size_t)j * n1,
                           wk + (size_t)j * n1, uptr(i) + (size_t)j * n1, 1, false);
    }
    ctx.sync();
    // D_i -= S_i U_i
    {
      const double *S = Sup(i);
      for (int e = tid; e < n0 * n0; e += NT_) {
        const int r = e % n0, c = e / n0;
        double acc = 0.0;
        if (S) {
          for (int k = 0; k < n1; ++k)
            acc += S[r + (size_t)k * n0] * uptr(i)[k + (size_t)c * n1];
        } else {
          acc = -uptr(i)[r + (size_t)c * n1];
        }
        bptr(i)[e] -= acc;
      }
    }
    ctx.sync();
  }
  if (ok && dm(0) > 0) {
    if (!bk_factor_group<8>(grp, bptr(0), dm(0), dm(0), dd_(0), sd_(0), pm_(0), kd_(0), pv))
      ok = false;
    else
      solve_vec(0, sol + off(0));
  }
  if (ok) {
    auto fwd_U = [&](double *v) { // v_{i+1} -= U_i v_i   (:130-133)
      for (int i = 0; i + 1 < NB; ++i) {
        const int n1 = dm(i + 1), n0 = dm(i);
        for (int r = tid; r < n1; r += NT_) {
          double acc = 0.0;
          for (int k = 0; k < n0; ++k)
            acc += uptr(i)[r + (size_t)k * n1] * v[off(i) + k];
          v[off(i + 1) + r] -= acc;
        }
        ctx.sync();
      }
    };
    fwd_U(sol);
    // ---- iterative refinement (parallel-solver.hxx:185-202)
    for (int it = 0; it < max_refine; ++it) {
      // err = rhs - A sol  (blockTridiagMatMul with the ORIGINAL blocks, block-tridiagonal.hpp:52-75)
      for (int b = 0; b < NB; ++b) {
        const int n = dm(b);
        const double *Do = Dorig(b);
        for (int i = tid; i < n; i += NT_) {
          double acc = 0.0;
          if (b > 0) { // sub-diagonal block = S_{b-1}^T
            const double *S = Sup(b - 1);
            const int c = dm(b - 1);
            if (S) {
              for (int k = 0; k < c; ++k)
                acc += S[k + (size_t)i * c] * sol[off(b - 1) + k];
            } else {
              acc += -sol[off(b - 1) + i];
            }
          }
          if (Do)
            for (int k = 0; k < n; ++k)
              acc += Do[i + (size_t)k * n] * sol[off(b) + k];
          if (b + 1 < NB) {
            const double *S = Sup(b);
            const int c = dm(b + 1);
            if (S) {
              for (int k = 0; k < c; ++k)
                acc += S[i + (size_t)k * n] * sol[off(b + 1) + k];
            } else {
              acc += -sol[off(b + 1) + i];
            }
          }
          err[off(b) + i] = rhs_at(b, i) - acc;
        }
      }
      ctx.sync();
      double resdl = 0.0; // infinity norm, computed redundantly by every thread
      for (int i = 0; i < TD; ++i)
        resdl = fmax(resdl, fabs(err[i]));
      if (!(resdl > thr)) // (NaN residuals stop the loop as well)
        break;
      // blockTridiagRefinementStep (block-tridiagonal.hpp:147-182)
      for (int i = NB - 2; i >= 0; --i) {
        solve_vec(i + 1, err + off(i + 1));
        sub_Sx(i, err + off(i), err + off(i + 1));
        ctx.sync();
      }
      solve_vec(0, err + off(0));
      fwd_U(err);
      for (int i = tid; i < TD; i += NT_)
        sol[i] += err[i];
      ctx.sync();
    }
  } else {
    st |= ST_CONDENSED_FACTOR_FAILED;
  }
  double *cond = p.cond + (size_t)inst * TD;
  for (int i = tid; i < TD; i += NT_)
    cond[i] = sol[i];
  for (int i = tid; i < nx + nc0; i += NT_) // kkt0.ff = [x_0; lbda_0]
    p.kkt0[(size_t)inst * (nx + nc0) + i] = (i < nx) ? sol[nc0 + i] : sol[i - nx];
  if (tid == 0) {
    if (st)
      ctx.atomic_or(p.status + inst, st);
    if (p.pivstat && pv)
      ctx.atomic_add(p.pivstat + inst, pv);
  }
  ctx.sync();
}

// collapseFeedback of the parallel solver (gar/parallel-solver.hpp:41-51): K_0 -= Kth_0 * sub[1],
// where after the swap of :180-181 sub[1] is the ORIGINAL sub-diagonal block Vxt_0^T.
template <class Ctx> AB2_D void collapse_feedback(Ctx &ctx, const SweepParams &p, const int nx, const int nu, const int nc, const int inst) {
  const int N = p.N, nr = nu + nc + nx, nth = nx;
  double *K = p.fb + (size_t)inst * N * nr * nx;
  const double *Kth = p.fth + (size_t)inst * N * nr * nth;
  const double *Vxt0 = p.Vxt + (size_t)inst * (N + 1) * nx * nth; // nx x nth column-major
  for (int e = ctx.tid; e < nu * nx; e += ctx.nthreads) {
    const int i = e / nx, j = e % nx;
    double acc = 0.0;
    for (int c = 0; c < nth; ++c)
      acc += Kth[i * nth + c] * Vxt0[j + (size_t)c * nx];
    K[i * nx + j] -= acc;
  }
}

} // namespace ab2
