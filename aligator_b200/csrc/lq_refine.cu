// lq_refine.cu -- the residual kernel of ab2_gar_refine, ab2_gar_refine_many and ab2_gar_kkt_error.  Refinement
// improves a solution estimate z of K z = -h on the last backward's factorisation, with resolve(r) = -K^-1 r
// (lq_resolve.cuh) as the correction solver and linear_step_kernel (linesearch.cu) as the update z += delta.  The update
// cannot be fused into the next residual launch: the residual of knot t reads x_{t+1} and lambda_t, which other warps
// would be updating.
//  * refine_residual_kernel: r = K z + h in resolve's rhs layouts, row by row (lambda_{t+1} = lams[t], lambda_t =
//    lams[t-1]):
//      q-row  Q x_t + S u_t + C^T v_t + A^T lambda_{t+1} - lambda_t + q_t     (t = 0: + G0^T lambda_0 instead of -lambda_0)
//      r-row  S^T x_t + R u_t + D^T v_t + B^T lambda_{t+1} + r_t
//      d-row  C x_t + D u_t - mu v_t + d_t
//      f-row  A x_t + B u_t - x_{t+1} + f_t
//      q_N    Q_N x_N + C_N^T v_N - lambda_N + q_N   (N = 0: + G0^T lambda_0),   d_N  C_N x_N - mu v_N + d_N,
//      g0     G0 x_0 + g0
//    Q and R are used as stored.  These are the rows of lqrComputeKktError (gar/utils.hxx:88-182).  With FAMILIES the
//    kernel keeps one maximum per row family, lqrComputeKktError's three norms: column col + 0 the f and g0 rows
//    (dynamics), col + 1 the d and d_N rows (constraints), col + 2 the q, r and q_N rows (stationarity).  That is
//    ab2_gar_kkt_error, with h the problem's own vectors and z the last forward pass.  Without it, one maximum of every
//    row in column col.  h is the problem's own vectors (read from the records) or a caller's right-hand sides.
//
// Layout of the residual kernel: one warp per group of K consecutive stage knots, grid-stride, with K = 32 / rows per
// knot (2 at C3, 1 at C2), so that short records leave few lanes idle.  A record of at most kTile doubles is staged
// in the warp's slice of shared memory by cp.async, double-buffered: the next group's records are in flight while
// the current group is summed.  Longer records (C5) are read in place.  The group's records are staged once and the
// warp loops over the right-hand sides.  The terminal and g0 rows get one warp per (instance, rhs).  Each row is
// summed by one lane in a fixed order, and the per-instance max |r| meets through an integer atomicMax on the bit
// pattern of a non-negative double (max is order-independent): right-hand side j's result is bit for bit
// independent of nrhs, of j's position and of timing.
#include <cuda_runtime.h>

#include "cp_async.cuh"
#include "lq_record.cuh"
#include "lq_refine.h"

namespace ab2 {

namespace {
constexpr int kWarps = 8;  // warps per CTA
constexpr int kTile = 512; // records of at most this many doubles are staged in shared memory

// row i of M y for the column-major m x n block M
__device__ __forceinline__ double rowdot(const double *M, int m, int n, int i, const double *y) {
  double s = 0.0;
  for (int c = 0; c < n; ++c)
    s = fma(M[i + c * m], y[c], s);
  return s;
}
// row i of M^T y (column i of M) for the column-major block M with m rows
__device__ __forceinline__ double coldot(const double *M, int m, int i, const double *y) {
  double s = 0.0;
  for (int r = 0; r < m; ++r)
    s = fma(M[i * m + r], y[r], s);
  return s;
}
// running infinity norm that keeps a NaN once it has seen one
__device__ __forceinline__ double upd(double m, double s) {
  const double v = fabs(s);
  return (v > m || v != v) ? v : m;
}
__device__ __forceinline__ double warp_max(double m) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    m = upd(m, __shfl_xor_sync(0xffffffffu, m, o));
  return m;
}
__device__ __forceinline__ void atomic_max_nonneg(double *addr, double v) {
  atomicMax(reinterpret_cast<unsigned long long *>(addr), (unsigned long long)__double_as_longlong(v));
}

// global address of stage record `it` = (b, t), through the ring head
__device__ __forceinline__ const double *record(const RefineResidualArgs &a, long it) {
  const int N = a.d.N;
  const long b = it / N;
  return a.stage + (b * N + ring_slot((int)(it - b * N), a.stage_head, N)) * a.d.srec;
}
// the records of the K knots of group g (fewer in the last group) to dst
__device__ __forceinline__ void issue(const RefineResidualArgs &a, int K, long nS, long g, double *dst, int lane) {
  const long k0 = g * K;
  const int kn = nS - k0 < K ? (int)(nS - k0) : K;
  for (int k = 0; k < kn; ++k)
    stage_copy(dst + k * a.d.srec, record(a, k0 + k), a.d.srec, lane);
}

int sm_count() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}
// knots per warp: as many as fit 32 lanes with one row each
int knots_per_warp(const AdjointDims &d) {
  const int nrow = 2 * d.nx + d.nu + d.nc;
  return nrow < 32 ? 32 / nrow : 1;
}
} // namespace

template <bool FAMILIES>
__global__ void __launch_bounds__(kWarps * 32, 2) refine_residual_kernel(const RefineResidualArgs a, int K, int staged,
                                                                       int warp_doubles) {
  extern __shared__ __align__(16) double smem[];
  const AdjointDims d = a.d;
  const int nx = d.nx, nu = d.nu, nc = d.nc, nct = d.nct, nc0 = d.nc0, N = d.N, B = d.batch, srec = d.srec;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int nrow = 2 * nx + nu + nc, nvec = 4 * nx + nu + nc; // vectors [x | u | v | l_{t+1} | l_t | x_{t+1}]
  // [records of the current group | records of the next group | vectors]; buffer `cur` at buf + cur * bstride
  const int bstride = staged ? K * srec : 0;
  double *const buf = smem + (size_t)wid * warp_doubles, *const vec = buf + 2 * bstride;
  const StageOffsets o = stage_offsets(nx, nu, nc);
  const long nS = (long)B * N, nG = N > 0 ? (nS + K - 1) / K : 0, nT = (long)B * a.nrhs;
  const long w0 = (long)blockIdx.x * kWarps + wid, ws = (long)gridDim.x * kWarps;
  // ---- stage knots, K per warp ----
  int cur = 0;
  if (staged && w0 < nG)
    issue(a, K, nS, w0, buf, lane);
  cp_commit();
  for (long g = w0; g < nG; g += ws) {
    if (staged && g + ws < nG)
      issue(a, K, nS, g + ws, buf + (cur ^ 1) * bstride, lane); // in flight while this group is summed
    cp_commit();
    cp_wait_prev();
    __syncwarp();
    const long k0 = g * K;
    const int kn = nS - k0 < K ? (int)(nS - k0) : K;
    const int klane = K > 1 ? lane / nrow : 0; // the knot of this lane's rows
    for (int j = 0; j < a.nrhs; ++j) {
      for (int p = lane; p < kn * nvec; p += 32) {
        const int k = p / nvec, e = p - k * nvec;
        const long it = k0 + k, b = it / N, t = it - b * N, jit = (long)j * nS + it, jb = (long)j * B + b;
        double v;
        if (e < nx)
          v = a.xs[(jit + jb) * nx + e];
        else if (e < nx + nu)
          v = a.us[jit * nu + e - nx];
        else if (e < nx + nu + nc)
          v = a.vs[jit * nc + e - nx - nu];
        else if (e < 2 * nx + nu + nc)
          v = a.lams[jit * nx + e - nx - nu - nc];
        else if (e < 3 * nx + nu + nc)
          v = t > 0 ? a.lams[(jit - 1) * nx + e - 2 * nx - nu - nc] : 0.0;
        else
          v = a.xs[(jit + jb + 1) * nx + e - 3 * nx - nu - nc];
        vec[p] = v;
      }
      __syncwarp();
      double m = 0.0, mc = 0.0, ms = 0.0; // FAMILIES: m the f rows, mc the d rows, ms the q and r rows
      for (int p = lane; p < kn * nrow; p += 32) {
        const int k = p / nrow, row = p - k * nrow;
        const long it = k0 + k, b = it / N, t = it - b * N, jit = (long)j * nS + it, jb = (long)j * B + b;
        const double *rec = staged ? buf + cur * bstride + k * srec : record(a, it);
        const double *x = vec + k * nvec, *u = x + nx, *v = u + nu, *ln = v + nc, *lp = ln + nx, *xn = lp + nx;
        double s;
        if (row < nx) {
          const int i = row;
          s = a.own ? rec[o.q + i] : (a.hq ? a.hq[(jit + jb) * nx + i] : 0.0);
          s += rowdot(rec + o.Q, nx, nx, i, x);
          s += rowdot(rec + o.S, nx, nu, i, u);
          s += coldot(rec + o.C, nc, i, v);
          s += coldot(rec + o.A, nx, i, ln);
          if (t > 0) {
            s -= lp[i];
          } else if (nc0 > 0) { // + G0^T lambda_0, G0 column-major [nc0][nx]
            const double *G = a.G0 + b * nc0 * nx, *l0 = a.lam0 + jb * nc0;
            s += coldot(G, nc0, i, l0);
          }
          if (a.q)
            a.q[(jit + jb) * nx + i] = s;
        } else if (row < nx + nu) {
          const int i = row - nx;
          s = a.own ? rec[o.r + i] : (a.hr ? a.hr[jit * nu + i] : 0.0);
          s += coldot(rec + o.S, nx, i, x);
          s += rowdot(rec + o.R, nu, nu, i, u);
          s += coldot(rec + o.D, nc, i, v);
          s += coldot(rec + o.B, nx, i, ln);
          if (a.r)
            a.r[jit * nu + i] = s;
        } else if (row < nx + nu + nc) {
          const int i = row - nx - nu;
          s = a.own ? rec[o.d + i] : (a.hd ? a.hd[jit * nc + i] : 0.0);
          s += rowdot(rec + o.C, nc, nx, i, x);
          s += rowdot(rec + o.D, nc, nu, i, u);
          s -= (a.mueq_b ? a.mueq_b[b] : a.mueq) * v[i];
          if (a.dv)
            a.dv[jit * nc + i] = s;
        } else {
          const int i = row - nx - nu - nc;
          s = a.own ? rec[o.f + i] : (a.hf ? a.hf[jit * nx + i] : 0.0);
          s += rowdot(rec + o.A, nx, nx, i, x);
          s += rowdot(rec + o.B, nx, nu, i, u);
          s -= xn[i];
          if (a.f)
            a.f[jit * nx + i] = s;
        }
        if constexpr (FAMILIES) {
          if (row < nx + nu)
            ms = upd(ms, s);
          else if (row < nx + nu + nc)
            mc = upd(mc, s);
          else
            m = upd(m, s);
        } else {
          m = upd(m, s);
        }
      }
      if (a.norms)
        for (int k = 0; k < kn; ++k) { // one maximum per knot of the group and family
          double mk[FAMILIES ? 3 : 1];   // the families' warp reductions overlap when no atomic sits between them
#pragma unroll
          for (int f = 0; f < (FAMILIES ? 3 : 1); ++f)
            mk[f] = warp_max(klane == k ? (f == 0 ? m : f == 1 ? mc : ms) : 0.0);
          if (lane == 0) {
            const long b = (k0 + k) / N;
#pragma unroll
            for (int f = 0; f < (FAMILIES ? 3 : 1); ++f)
              atomic_max_nonneg(a.norms + ((long)j * B + b) * a.nstride + a.col + f, mk[f]);
          }
        }
      __syncwarp(); // the vectors are overwritten next
    }
    cur ^= 1;
  }
  cp_wait_all();
  // ---- (instance b, rhs j): rows [q_N (nx) | d_N (nct) | g0 (nc0)] ----
  const TermOffsets to = term_offsets(nx, nct);
  const int trows = nx + nct + nc0;
  for (long jb = w0; jb < nT; jb += ws) {
    const long b = jb % B;
    const double *T = a.term + b * d.trec, *G = a.G0 + b * nc0 * nx;
    const double *x = a.xs + (jb * (N + 1) + N) * nx, *vT = a.vsT + jb * nct, *x0 = a.xs + jb * (N + 1) * nx;
    const double *l0 = a.lam0 + jb * nc0, *lN = N > 0 ? a.lams + (jb * N + N - 1) * nx : nullptr;
    double m = 0.0, mc = 0.0, ms = 0.0; // FAMILIES: m the g0 rows, mc the d_N rows, ms the q_N rows
    for (int row = lane; row < trows; row += 32) {
      double s;
      if (row < nx) {
        const int i = row;
        s = a.own ? T[to.q + i] : (a.hq ? a.hq[(jb * (N + 1) + N) * nx + i] : 0.0);
        s += rowdot(T + to.Q, nx, nx, i, x);
        s += coldot(T + to.C, nct, i, vT);
        if (N > 0)
          s -= lN[i];
        else if (nc0 > 0) // x_0 = x_N: + G0^T lambda_0
          s += coldot(G, nc0, i, l0);
        if (a.q)
          a.q[(jb * (N + 1) + N) * nx + i] = s;
      } else if (row < nx + nct) {
        const int i = row - nx;
        s = a.own ? T[to.d + i] : (a.hdN ? a.hdN[jb * nct + i] : 0.0);
        s += rowdot(T + to.C, nct, nx, i, x);
        s -= (a.mueq_b ? a.mueq_b[b] : a.mueq) * vT[i];
        if (a.dN)
          a.dN[jb * nct + i] = s;
      } else {
        const int i = row - nx - nct;
        s = a.own ? a.g0[b * nc0 + i] : (a.hg0 ? a.hg0[jb * nc0 + i] : 0.0);
        s += rowdot(G, nc0, nx, i, x0);
        if (a.g0out)
          a.g0out[jb * nc0 + i] = s;
      }
      if constexpr (FAMILIES) {
        if (row < nx)
          ms = upd(ms, s);
        else if (row < nx + nct)
          mc = upd(mc, s);
        else
          m = upd(m, s);
      } else {
        m = upd(m, s);
      }
    }
    if (a.norms) {
      double mk[FAMILIES ? 3 : 1];
#pragma unroll
      for (int f = 0; f < (FAMILIES ? 3 : 1); ++f)
        mk[f] = warp_max(f == 0 ? m : f == 1 ? mc : ms);
      if (lane == 0) {
#pragma unroll
        for (int f = 0; f < (FAMILIES ? 3 : 1); ++f)
          atomic_max_nonneg(a.norms + jb * a.nstride + a.col + f, mk[f]);
      }
    }
  }
}

cudaError_t launch_refine_residual(const RefineResidualArgs &a, bool families, cudaStream_t st) {
  const AdjointDims &d = a.d;
  const int K = knots_per_warp(d);
  const long nG = d.N > 0 ? ((long)d.batch * d.N + K - 1) / K : 0, items = nG + (long)d.batch * a.nrhs;
  if (a.nrhs <= 0 || items <= 0)
    return cudaSuccess;
  const int staged = d.N > 0 && d.srec <= kTile;
  const int nvec = 4 * d.nx + d.nu + d.nc;
  const int warp_doubles = ((staged ? 2 * K * d.srec : 0) + K * nvec + 1) & ~1; // (srec is even)
  const size_t smem = (size_t)warp_doubles * kWarps * sizeof(double);
  const auto kernel = families ? refine_residual_kernel<true> : refine_residual_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess)
    return e;
  int per_sm = 1;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kWarps * 32, smem);
  if (e != cudaSuccess)
    return e;
  long grid = (items + kWarps - 1) / kWarps;
  const long full = (long)sm_count() * (per_sm > 0 ? per_sm : 1);
  grid = grid < full ? grid : full;
  kernel<<<(int)grid, kWarps * 32, smem, st>>>(a, K, staged, warp_doubles);
  return cudaGetLastError();
}

} // namespace ab2
