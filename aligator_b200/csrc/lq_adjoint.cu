// lq_adjoint.cu -- the records kernel of ab2_gar_adjoint and ab2_gar_tangent.
//
// The LQ solve is the solution of one symmetric KKT system K z = -h.  The gradient of a loss with cotangent zbar
// needs w = K^-1 zbar, and the tangent along (Kdot, hdot) is zdot = -K^-1 rho with rho = Kdot z + hdot: each is the
// same LQ problem with new vectors, which the existing sweep kernels solve unchanged.  adjoint_records_kernel builds
// that problem: every matrix block copied from the current records, the vectors q, r, d, f (and q_N, d_N, g0)
// replaced by minus the cotangent (adjoint) or by rho (tangent, copy).  The gradients and rho are the Jacobian
// kernels' (lq_jacobian.cu) at nrhs = 1.
//
// Pure streaming work (HBM-bound), built like lq_assemble.cu: one element per thread over the contiguous
// [batch][N][record] arrays, grid-stride over 8 CTAs of 256 threads per SM, with the map
// "element of the record -> (block, row)" built once per CTA in shared memory, so that loads of the records and
// stores of the outputs are coalesced.
#include <cuda_runtime.h>

#include "lq_adjoint.h"
#include "lq_record.cuh"

namespace ab2 {

namespace {
// adjoint records: what element e of a stage record holds
enum : int { R_COPY = 0, R_X = 1, R_U = 2, R_V = 3, R_L = 4, R_PAD = 5 };

// a vector entry of the new problem: -p[i] (NULL = zero cotangent), or p[i] itself with copy
__device__ __forceinline__ double vec(const double *p, long i, bool copy) {
  if (copy)
    return p[i];
  return -(p ? p[i] : 0.0);
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
  extern __shared__ int lut[]; // [srec]: kind | row << 4
  const AdjointDims d = a.d;
  const int nx = d.nx, nu = d.nu, nc = d.nc, N = d.N;
  const StageOffsets so = stage_offsets(nx, nu, nc);
  for (int e = threadIdx.x; e < d.srec; e += blockDim.x) {
    const RecElem el = stage_elem(so, nx, nu, nc, e);
    int k;
    switch (el.blk) {
    case BK_F: k = R_L; break;  // f <- -lambdabar_{t+1}
    case BK_QV: k = R_X; break; // q <- -xbar_t
    case BK_RV: k = R_U; break; // r <- -ubar_t
    case BK_DV: k = R_V; break; // d <- -vbar_t
    case BK_PAD: k = R_PAD; break;
    default: k = R_COPY;        // A, B, Q, S, R, C, D
    }
    lut[e] = k | (el.row << 4);
  }
  __syncthreads();
  const TermOffsets to = term_offsets(nx, d.nct);
  const long nS = (long)d.batch * N * d.srec, nT = (long)d.batch * d.trec, ng = (long)d.batch * d.nc0;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < nS + nT + ng; i += (long)gridDim.x * blockDim.x) {
    if (i < nS) {
      const long rec = i / d.srec;
      const int e = (int)(i - rec * d.srec);
      const long b = rec / N;
      const int t = (int)(rec - b * N), ent = lut[e], o = ent >> 4;
      double v;
      switch (ent & 15) {
      case R_COPY: v = a.stage[(b * N + ring_slot(t, a.stage_head, N)) * d.srec + e]; break; // (cycle_append)
      case R_X: v = vec(a.xs, (b * (N + 1) + t) * nx + o, a.copy); break;
      case R_U: v = vec(a.us, rec * nu + o, a.copy); break;
      case R_V: v = vec(a.vs, rec * nc + o, a.copy); break;
      case R_L: v = vec(a.lams, rec * nx + o, a.copy); break;
      default: v = 0.0;
      }
      a.adj_stage[i] = v;
    } else if (i < nS + nT) { // terminal [Q | q | C | d]
      const long j = i - nS, b = j / d.trec;
      const RecElem el = term_elem(to, nx, d.nct, (int)(j - b * d.trec));
      double v;
      if (el.blk == BK_QV)
        v = vec(a.xs, (b * (N + 1) + N) * nx + el.row, a.copy);
      else if (el.blk == BK_DV)
        v = vec(a.vsT, b * d.nct + el.row, a.copy);
      else
        v = a.term[j];
      a.adj_term[j] = v;
    } else {
      const long j = i - nS - nT;
      a.adj_g0[j] = vec(a.lam0, j, a.copy);
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

} // namespace ab2
