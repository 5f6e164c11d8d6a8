// lq_theta.cu -- the kernels of ab2_gar_theta_tangent and ab2_gar_theta_adjoint: the programs of lq_theta.cuh on one
// warp per work item.
#include <cuda_runtime.h>

#include "item_launch.cuh"
#include "lq_theta.h"

namespace ab2 {

namespace {
constexpr int kMaxChunk = 32; // directions one warp holds on chip

template <bool ADJ>
__global__ void __launch_bounds__(kItemMaxWarps * 32) theta_kernel(const ThetaArgs a, int item_doubles, long items,
                                                                   int chunks) {
  extern __shared__ __align__(16) double smem[];
  const int wid = threadIdx.x >> 5;
  const long item = (long)blockIdx.x * (blockDim.x >> 5) + wid;
  if (item >= items)
    return;
  const long b = item / chunks;
  const int j0 = (int)(item - b * chunks) * a.chunk;
  const int R = a.nrhs - j0 < a.chunk ? a.nrhs - j0 : a.chunk;
  const ItemWarpCtx ctx{(int)(threadIdx.x & 31), 32};
  double *sm = smem + (size_t)wid * item_doubles;
  if (ADJ)
    theta_adjoint_item(a, ctx, sm, b, j0, R);
  else
    theta_tangent_item(a, ctx, sm, b, j0, R);
}

template <bool ADJ> cudaError_t launch(ThetaArgs a, cudaStream_t st) {
  if (a.nrhs <= 0 || a.batch <= 0)
    return cudaSuccess;
  auto bytes = [&](int chunk) {
    return (size_t)theta_item_doubles(a.nx, a.nu, a.nc, a.nct, a.nc0, a.nth, chunk) * sizeof(double);
  };
  int chunk = a.nrhs < kMaxChunk ? a.nrhs : kMaxChunk;
  while (chunk > 1 && bytes(chunk) > kThetaSmemMax)
    chunk /= 2;
  a.chunk = chunk;
  const size_t item_bytes = bytes(chunk);
  if (item_bytes > kThetaSmemMax)
    return cudaErrorInvalidValue;
  const int wpc = item_warps_per_cta(item_bytes);
  const size_t smem = item_bytes * wpc;
  cudaError_t e = cudaFuncSetAttribute(theta_kernel<ADJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess)
    return e;
  const int chunks = (a.nrhs + chunk - 1) / chunk;
  const long items = (long)a.batch * chunks;
  const long grid = (items + wpc - 1) / wpc;
  theta_kernel<ADJ><<<(unsigned)grid, wpc * 32, smem, st>>>(a, (int)(item_bytes / sizeof(double)), items, chunks);
  return cudaGetLastError();
}
} // namespace

cudaError_t launch_theta_tangent(ThetaArgs a, cudaStream_t st) { return launch<false>(a, st); }
cudaError_t launch_theta_adjoint(ThetaArgs a, cudaStream_t st) { return launch<true>(a, st); }

} // namespace ab2
