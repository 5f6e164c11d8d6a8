// lq_factor_adjoint.cu -- the kernels of ab2_gar_factor_adjoint: the program of lq_factor_adjoint.cuh on one warp per
// instance, or on one whole CTA per instance when the item's shared memory leaves room for no other (config 5).
#include <cuda_runtime.h>

#include "item_launch.cuh"
#include "lq_factor_adjoint.h"

namespace ab2 {

__global__ void __launch_bounds__(kItemMaxWarps * 32) factor_adjoint_warp_kernel(const FactorAdjointArgs a,
                                                                                int item_doubles) {
  extern __shared__ __align__(16) double smem[];
  const int wid = threadIdx.x >> 5;
  const long b = (long)blockIdx.x * (blockDim.x >> 5) + wid;
  if (b >= a.fac.batch)
    return;
  const ItemWarpCtx ctx{(int)(threadIdx.x & 31), 32};
  factor_adjoint_item(a, ctx, smem + (size_t)wid * item_doubles, b);
}

__global__ void __launch_bounds__(kItemCtaThreads, 1) factor_adjoint_cta_kernel(const FactorAdjointArgs a) {
  extern __shared__ __align__(16) double smem[];
  const ItemCtaCtx ctx{(int)threadIdx.x, (int)blockDim.x};
  factor_adjoint_item(a, ctx, smem, (long)blockIdx.x);
}

cudaError_t launch_factor_adjoint(const FactorAdjointArgs &a, cudaStream_t st) {
  if (a.fac.batch <= 0)
    return cudaSuccess;
  const size_t item_bytes = (size_t)factor_adjoint_item_doubles(a.fac.nx, a.fac.nu, a.fac.nc) * sizeof(double);
  if (item_bytes > kFactorAdjointSmemMax)
    return cudaErrorInvalidValue;
  return launch_items(factor_adjoint_warp_kernel, factor_adjoint_cta_kernel, a, a.fac.batch, item_bytes, st);
}

} // namespace ab2
