// lq_adjoint.cu -- the two streaming kernels around the adjoint sweep of ab2_gar_adjoint.
//
// The LQ solve is the solution of one symmetric KKT system K z = -h.  The gradient of a loss with cotangent zbar
// needs w = K^-1 zbar, which is the same LQ problem with new vectors; the existing sweep kernels solve it unchanged.
//  * adjoint_records_kernel builds that problem: every matrix block copied from the current records, the vectors
//    q, r, d, f (and q_N, d_N, g0) replaced by minus the cotangent.
//  * adjoint_grad_kernel turns (z, w) into gradient records in the problem's own layout:
//    dh = -w and dK = -w z^T, read out of K's blocks (the symmetric Q and R get the symmetric part).
//
// Pure streaming work (HBM-bound), built like lq_assemble.cu: one element per thread over the contiguous
// [batch][N][record] arrays, grid-stride over 8 CTAs of 256 threads per SM, with the map
// "element of the record -> (block, row, column)" built once per CTA in shared memory, so that loads of the
// records and stores of the outputs are coalesced.
#include <cuda_runtime.h>

#include "lq_adjoint.h"

namespace ab2 {

namespace {
// adjoint records: what element e of a stage record holds
enum : int { R_COPY = 0, R_X = 1, R_U = 2, R_V = 3, R_L = 4, R_PAD = 5 };
// gradient records: the vectors a block's gradient is made of
enum : unsigned { V_X = 0, V_U = 1, V_V = 2, V_L = 3 };               // x_t, u_t, v_t, lambda_{t+1}
enum : unsigned { M_PAIR = 0, M_HALF = 1, M_SINGLE = 2, M_ZERO = 3 }; // -(a b' + a' b), half of it, -a, 0

__device__ __forceinline__ double neg(const double *p, long i) { return -(p ? p[i] : 0.0); } // NULL = zero cotangent

__device__ __forceinline__ unsigned grad_entry(unsigned ai, unsigned bj, unsigned mode, int i, int j) {
  return ai | (bj << 2) | (mode << 4) | ((unsigned)i << 8) | ((unsigned)j << 20);
}
__device__ __forceinline__ const double *pick(unsigned k, const double *x, const double *u, const double *v,
                                              const double *l) {
  return k == V_X ? x : k == V_U ? u : k == V_V ? v : l;
}
// one gradient element from its map entry: P = primal vectors, W = adjoint vectors of the knot
__device__ __forceinline__ double grad_value(unsigned ent, const double *px, const double *pu, const double *pv,
                                             const double *pl, const double *wx, const double *wu, const double *wv,
                                             const double *wl) {
  const unsigned ai = ent & 3, bj = (ent >> 2) & 3, mode = (ent >> 4) & 3;
  const int i = (int)((ent >> 8) & 0xfff), j = (int)(ent >> 20);
  if (mode == M_ZERO)
    return 0.0;
  const double wa = pick(ai, wx, wu, wv, wl)[i];
  if (mode == M_SINGLE)
    return -wa;
  const double s = wa * pick(bj, px, pu, pv, pl)[j] + pick(ai, px, pu, pv, pl)[i] * pick(bj, wx, wu, wv, wl)[j];
  return mode == M_HALF ? -(0.5 * s) : -s;
}

long grid_for(long total) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  long grid = (total + 255) / 256;
  if (grid > (long)sms * 8)
    grid = (long)sms * 8;
  return grid > 0 ? grid : 1;
}
} // namespace

__global__ void __launch_bounds__(256) adjoint_records_kernel(const AdjointRecordArgs a) {
  extern __shared__ int lut[]; // [srec]: kind | offset << 4
  const AdjointDims d = a.d;
  const int nx = d.nx, nu = d.nu, nc = d.nc, N = d.N, nxx = nx * nx, nxu = nx * nu;
  for (int e = threadIdx.x; e < d.srec; e += blockDim.x) {
    int r = e, k;
    if (r < nxx + nxu) { // A, B
      k = R_COPY;
    } else if ((r -= nxx + nxu) < nx) { // f <- -lambdabar_{t+1}
      k = R_L;
    } else if ((r -= nx) < nxx + nxu + nu * nu) { // Q, S, R
      k = R_COPY;
    } else if ((r -= nxx + nxu + nu * nu) < nx) { // q <- -xbar_t
      k = R_X;
    } else if ((r -= nx) < nu) { // r <- -ubar_t
      k = R_U;
    } else if ((r -= nu) < nc * (nx + nu)) { // C, D
      k = R_COPY;
    } else if ((r -= nc * (nx + nu)) < nc) { // d <- -vbar_t
      k = R_V;
    } else {
      k = R_PAD;
    }
    lut[e] = k | (r << 4);
  }
  __syncthreads();
  const long nS = (long)d.batch * N * d.srec, nT = (long)d.batch * d.trec, ng = (long)d.batch * d.nc0;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < nS + nT + ng; i += (long)gridDim.x * blockDim.x) {
    if (i < nS) {
      const long rec = i / d.srec;
      const int e = (int)(i - rec * d.srec);
      const long b = rec / N;
      const int t = (int)(rec - b * N), ent = lut[e], o = ent >> 4;
      double v;
      switch (ent & 15) {
      case R_COPY: { // the current record, read through the ring head (cycle_append)
        const int slot = t + a.stage_head >= N ? t + a.stage_head - N : t + a.stage_head;
        v = a.stage[(b * N + slot) * d.srec + e];
        break;
      }
      case R_X: v = neg(a.xs, (b * (N + 1) + t) * nx + o); break;
      case R_U: v = neg(a.us, rec * nu + o); break;
      case R_V: v = neg(a.vs, rec * nc + o); break;
      case R_L: v = neg(a.lams, rec * nx + o); break;
      default: v = 0.0;
      }
      a.adj_stage[i] = v;
    } else if (i < nS + nT) { // terminal [Q | q | C | d]
      const long j = i - nS, b = j / d.trec;
      const int e = (int)(j - b * d.trec);
      double v;
      if (e < nxx || (e >= nxx + nx && e < nxx + nx + d.nct * nx))
        v = a.term[j];
      else if (e < nxx + nx)
        v = neg(a.xs, (b * (N + 1) + N) * nx + (e - nxx));
      else
        v = neg(a.vsT, b * d.nct + (e - nxx - nx - d.nct * nx));
      a.adj_term[j] = v;
    } else {
      const long j = i - nS - nT;
      a.adj_g0[j] = neg(a.lam0, j);
    }
  }
}

__global__ void __launch_bounds__(256) adjoint_grad_kernel(const AdjointGradArgs a) {
  extern __shared__ unsigned map[]; // [srec] stage entries, then [trec] terminal entries
  const AdjointDims d = a.d;
  const int nx = d.nx, nu = d.nu, nc = d.nc, nct = d.nct, nc0 = d.nc0, N = d.N, nxx = nx * nx, nxu = nx * nu;
  for (int e = threadIdx.x; e < d.srec; e += blockDim.x) {
    int r = e;
    unsigned ent;
    if (r < nxx) // dA = -(lt x^T + l xt^T)
      ent = grad_entry(V_L, V_X, M_PAIR, r % nx, r / nx);
    else if ((r -= nxx) < nxu) // dB = -(lt u^T + l ut^T)
      ent = grad_entry(V_L, V_U, M_PAIR, r % nx, r / nx);
    else if ((r -= nxu) < nx) // df = -lt
      ent = grad_entry(V_L, 0, M_SINGLE, r, 0);
    else if ((r -= nx) < nxx) // dQ = -1/2 (xt x^T + x xt^T)
      ent = grad_entry(V_X, V_X, M_HALF, r % nx, r / nx);
    else if ((r -= nxx) < nxu) // dS = -(xt u^T + x ut^T)
      ent = grad_entry(V_X, V_U, M_PAIR, r % nx, r / nx);
    else if ((r -= nxu) < nu * nu) // dR = -1/2 (ut u^T + u ut^T)
      ent = grad_entry(V_U, V_U, M_HALF, r % nu, r / nu);
    else if ((r -= nu * nu) < nx) // dq = -xt
      ent = grad_entry(V_X, 0, M_SINGLE, r, 0);
    else if ((r -= nx) < nu) // dr = -ut
      ent = grad_entry(V_U, 0, M_SINGLE, r, 0);
    else if ((r -= nu) < nc * nx) // dC = -(vt x^T + v xt^T)
      ent = grad_entry(V_V, V_X, M_PAIR, r % nc, r / nc);
    else if ((r -= nc * nx) < nc * nu) // dD = -(vt u^T + v ut^T)
      ent = grad_entry(V_V, V_U, M_PAIR, r % nc, r / nc);
    else if ((r -= nc * nu) < nc) // dd = -vt
      ent = grad_entry(V_V, 0, M_SINGLE, r, 0);
    else
      ent = grad_entry(0, 0, M_ZERO, 0, 0);
    map[e] = ent;
  }
  for (int e = threadIdx.x; e < d.trec; e += blockDim.x) { // terminal [Q | q | C | d] with x = x_N, v = v_N
    int r = e;
    unsigned ent;
    if (r < nxx)
      ent = grad_entry(V_X, V_X, M_HALF, r % nx, r / nx);
    else if ((r -= nxx) < nx)
      ent = grad_entry(V_X, 0, M_SINGLE, r, 0);
    else if ((r -= nx) < nct * nx)
      ent = grad_entry(V_V, V_X, M_PAIR, r % nct, r / nct);
    else
      ent = grad_entry(V_V, 0, M_SINGLE, r - nct * nx, 0);
    map[d.srec + e] = ent;
  }
  __syncthreads();
  // outputs that are NULL take no part in the index space
  const long nS = a.stage ? (long)d.batch * N * d.srec : 0, nT = a.term ? (long)d.batch * d.trec : 0;
  const long nG = a.G0 ? (long)d.batch * nc0 * nx : 0, ng = a.g0 ? (long)d.batch * nc0 : 0;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < nS + nT + nG + ng; i += (long)gridDim.x * blockDim.x) {
    if (i < nS) {
      const long rec = i / d.srec;
      const int e = (int)(i - rec * d.srec);
      const long b = rec / N, xo = (rec + b) * nx; // x_t of knot (b, t): row b (N + 1) + t
      a.stage[i] = grad_value(map[e], a.xs + xo, a.us + rec * nu, a.vs + rec * nc, a.lams + rec * nx, a.wxs + xo,
                              a.wus + rec * nu, a.wvs + rec * nc, a.wlams + rec * nx);
    } else if (i < nS + nT) {
      const long j = i - nS, b = j / d.trec, xo = (b * (N + 1) + N) * nx;
      a.term[j] = grad_value(map[d.srec + (int)(j - b * d.trec)], a.xs + xo, nullptr, a.vsT + b * nct, nullptr,
                             a.wxs + xo, nullptr, a.wvsT + b * nct, nullptr);
    } else if (i < nS + nT + nG) { // dG0 = -(lt_0 x_0^T + l_0 xt_0^T), column-major [nc0][nx]
      const long j = i - nS - nT, b = j / ((long)nc0 * nx);
      const int e = (int)(j - b * nc0 * nx), r = e % nc0, c = e / nc0;
      const long xo = b * (N + 1) * nx;
      a.G0[j] = -(a.wlam0[b * nc0 + r] * a.xs[xo + c] + a.lam0[b * nc0 + r] * a.wxs[xo + c]);
    } else { // dg0 = -lt_0
      const long j = i - nS - nT - nG;
      a.g0[j] = -a.wlam0[j];
    }
  }
}

cudaError_t launch_adjoint_records(const AdjointRecordArgs &a, cudaStream_t st) {
  const long total = (long)a.d.batch * a.d.N * a.d.srec + (long)a.d.batch * a.d.trec + (long)a.d.batch * a.d.nc0;
  const size_t smem = (size_t)(a.d.srec > 0 ? a.d.srec : 1) * sizeof(int);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(adjoint_records_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess)
      return e;
  }
  adjoint_records_kernel<<<(int)grid_for(total), 256, smem, st>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_adjoint_grad(const AdjointGradArgs &a, cudaStream_t st) {
  const AdjointDims &d = a.d;
  const long total = (a.stage ? (long)d.batch * d.N * d.srec : 0) + (a.term ? (long)d.batch * d.trec : 0) +
                     (a.G0 ? (long)d.batch * d.nc0 * d.nx : 0) + (a.g0 ? (long)d.batch * d.nc0 : 0);
  const size_t smem = (size_t)(d.srec + d.trec) * sizeof(unsigned);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(adjoint_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess)
      return e;
  }
  adjoint_grad_kernel<<<(int)grid_for(total), 256, smem, st>>>(a);
  return cudaGetLastError();
}

} // namespace ab2
