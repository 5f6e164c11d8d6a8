// lq_items.cu -- the kernels of the per-item programs: resolve (lq_resolve.cuh) and the θ tangent and adjoint
// (lq_theta.cuh) on one warp per (instance, chunk); the factorisation's adjoint (lq_factor_adjoint.cuh) and tangent
// (lq_factor_tangent.cuh) on one warp per instance, or on one whole CTA per instance when the item's shared memory
// leaves room for no other (config 5).
#include <cuda_runtime.h>

#include "item_launch.cuh"
#include "lq_items.h"

namespace ab2 {

__global__ void __launch_bounds__(kItemMaxWarps * 32) resolve_kernel(const ResolveArgs a, int item_doubles,
                                                                     long items, int chunks) {
  run_chunk_item(a, item_doubles, items, chunks, [&](const ItemWarpCtx &ctx, double *sm, long b, int j0, int R) {
    resolve_item(a, ctx, sm, b, j0, R);
  });
}

namespace {
template <bool ADJ>
__global__ void __launch_bounds__(kItemMaxWarps * 32) theta_kernel(const ThetaArgs a, int item_doubles, long items,
                                                                   int chunks) {
  run_chunk_item(a, item_doubles, items, chunks, [&](const ItemWarpCtx &ctx, double *sm, long b, int j0, int R) {
    if (ADJ)
      theta_adjoint_item(a, ctx, sm, b, j0, R);
    else
      theta_tangent_item(a, ctx, sm, b, j0, R);
  });
}
} // namespace

__global__ void __launch_bounds__(kItemMaxWarps * 32) factor_adjoint_warp_kernel(const FactorAdjointArgs a,
                                                                                int item_doubles) {
  run_warp_item(item_doubles, a.fac.batch,
                [&](const ItemWarpCtx &ctx, double *sm, long b) { factor_adjoint_item(a, ctx, sm, b); });
}

__global__ void __launch_bounds__(kItemCtaThreads, 1) factor_adjoint_cta_kernel(const FactorAdjointArgs a) {
  extern __shared__ __align__(16) double smem[];
  const ItemCtaCtx ctx{(int)threadIdx.x, (int)blockDim.x};
  factor_adjoint_item(a, ctx, smem, (long)blockIdx.x);
}

__global__ void __launch_bounds__(kItemMaxWarps * 32) factor_tangent_warp_kernel(const FactorTangentArgs a,
                                                                                int item_doubles) {
  run_warp_item(item_doubles, a.fac.batch,
                [&](const ItemWarpCtx &ctx, double *sm, long b) { factor_tangent_item(a, ctx, sm, b); });
}

__global__ void __launch_bounds__(kItemCtaThreads, 1) factor_tangent_cta_kernel(const FactorTangentArgs a) {
  extern __shared__ __align__(16) double smem[];
  const ItemCtaCtx ctx{(int)threadIdx.x, (int)blockDim.x};
  factor_tangent_item(a, ctx, smem, (long)blockIdx.x);
}

cudaError_t launch_resolve(ResolveArgs a, cudaStream_t st) {
  return launch_chunked_items(resolve_kernel, a, [&](int chunk) {
    return (size_t)resolve_item_doubles(a.nx, a.nu, a.nc, a.nc0, chunk) * sizeof(double);
  }, st);
}

static size_t theta_item_bytes(const ThetaArgs &a, int chunk) {
  return (size_t)theta_item_doubles(a.nx, a.nu, a.nc, a.nct, a.nc0, a.nth, chunk) * sizeof(double);
}
cudaError_t launch_theta_tangent(ThetaArgs a, cudaStream_t st) {
  return launch_chunked_items(theta_kernel<false>, a, [&](int chunk) { return theta_item_bytes(a, chunk); }, st);
}
cudaError_t launch_theta_adjoint(ThetaArgs a, cudaStream_t st) {
  return launch_chunked_items(theta_kernel<true>, a, [&](int chunk) { return theta_item_bytes(a, chunk); }, st);
}

cudaError_t launch_factor_adjoint(const FactorAdjointArgs &a, cudaStream_t st) {
  const size_t item_bytes = (size_t)factor_adjoint_item_doubles(a.fac.nx, a.fac.nu, a.fac.nc) * sizeof(double);
  return launch_items(factor_adjoint_warp_kernel, factor_adjoint_cta_kernel, a, a.fac.batch, item_bytes, st);
}

cudaError_t launch_factor_tangent(const FactorTangentArgs &a, cudaStream_t st) {
  const size_t item_bytes = (size_t)factor_tangent_item_doubles(a.fac.nx, a.fac.nu, a.fac.nc) * sizeof(double);
  return launch_items(factor_tangent_warp_kernel, factor_tangent_cta_kernel, a, a.fac.batch, item_bytes, st);
}

} // namespace ab2
