// lq_factor_adjoint.cu -- the kernels of ab2_gar_factor_adjoint: the program of lq_factor_adjoint.cuh on one warp per
// instance, or on one whole CTA per instance when the item's shared memory leaves room for no other (config 5).
#include <cuda_runtime.h>

#include "lq_factor_adjoint.h"

namespace ab2 {

namespace {
constexpr int kMaxWarps = 4;          // warps (independent items) per CTA
constexpr int kCtaBudget = 96 * 1024; // shared-memory bytes a CTA of warp items aims for; larger items take a CTA
constexpr int kCtaThreads = 256;      // lanes of one CTA-wide item

struct WarpCtx {
  int lane, nl;
  __device__ __forceinline__ void sync() const { __syncwarp(); }
};
struct CtaCtx {
  int lane, nl;
  __device__ __forceinline__ void sync() const { __syncthreads(); }
};
} // namespace

__global__ void __launch_bounds__(kMaxWarps * 32) factor_adjoint_warp_kernel(const FactorAdjointArgs a,
                                                                            int item_doubles) {
  extern __shared__ __align__(16) double smem[];
  const int wid = threadIdx.x >> 5;
  const long b = (long)blockIdx.x * (blockDim.x >> 5) + wid;
  if (b >= a.fac.batch)
    return;
  const WarpCtx ctx{(int)(threadIdx.x & 31), 32};
  factor_adjoint_item(a, ctx, smem + (size_t)wid * item_doubles, b);
}

__global__ void __launch_bounds__(kCtaThreads, 1) factor_adjoint_cta_kernel(const FactorAdjointArgs a) {
  extern __shared__ __align__(16) double smem[];
  const CtaCtx ctx{(int)threadIdx.x, (int)blockDim.x};
  factor_adjoint_item(a, ctx, smem, (long)blockIdx.x);
}

cudaError_t launch_factor_adjoint(const FactorAdjointArgs &a, cudaStream_t st) {
  if (a.fac.batch <= 0)
    return cudaSuccess;
  const size_t item_bytes = (size_t)factor_adjoint_item_doubles(a.fac.nx, a.fac.nu, a.fac.nc) * sizeof(double);
  if (item_bytes > kFactorAdjointSmemMax)
    return cudaErrorInvalidValue;
  cudaError_t e;
  if (item_bytes > kCtaBudget) {
    e = cudaFuncSetAttribute(factor_adjoint_cta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)item_bytes);
    if (e != cudaSuccess)
      return e;
    factor_adjoint_cta_kernel<<<(unsigned)a.fac.batch, kCtaThreads, item_bytes, st>>>(a);
    return cudaGetLastError();
  }
  int wpc = (int)(kCtaBudget / item_bytes);
  wpc = wpc < 1 ? 1 : (wpc > kMaxWarps ? kMaxWarps : wpc);
  const size_t smem = item_bytes * wpc;
  e = cudaFuncSetAttribute(factor_adjoint_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess)
    return e;
  const long grid = ((long)a.fac.batch + wpc - 1) / wpc;
  factor_adjoint_warp_kernel<<<(unsigned)grid, wpc * 32, smem, st>>>(a, (int)(item_bytes / sizeof(double)));
  return cudaGetLastError();
}

} // namespace ab2
