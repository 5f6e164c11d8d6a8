// lq_resolve.cu -- the kernel of ab2_gar_resolve: the program of lq_resolve.cuh on one warp per work item.
#include <cuda_runtime.h>

#include "lq_resolve.h"

namespace ab2 {

namespace {
constexpr int kMaxChunk = 32;          // right-hand sides one warp holds on chip
constexpr int kMaxWarps = 4;           // warps (independent items) per CTA
constexpr int kCtaBudget = 96 * 1024;  // shared-memory bytes a CTA aims for when it holds several items

struct WarpCtx {
  int lane, nl;
  __device__ __forceinline__ void sync() const { __syncwarp(); }
};
} // namespace

__global__ void __launch_bounds__(kMaxWarps * 32) resolve_kernel(const ResolveArgs a, int item_doubles, long items,
                                                                 int chunks) {
  extern __shared__ __align__(16) double smem[];
  const int wid = threadIdx.x >> 5;
  const long item = (long)blockIdx.x * (blockDim.x >> 5) + wid;
  if (item >= items)
    return;
  const long b = item / chunks;
  const int j0 = (int)(item - b * chunks) * a.chunk;
  const int R = a.nrhs - j0 < a.chunk ? a.nrhs - j0 : a.chunk;
  const WarpCtx ctx{(int)(threadIdx.x & 31), 32};
  resolve_item(a, ctx, smem + (size_t)wid * item_doubles, b, j0, R);
}

cudaError_t launch_resolve(ResolveArgs a, cudaStream_t st) {
  if (a.nrhs <= 0 || a.batch <= 0)
    return cudaSuccess;
  int chunk = a.nrhs < kMaxChunk ? a.nrhs : kMaxChunk;
  while (chunk > 1 && (size_t)resolve_item_doubles(a.nx, a.nu, a.nc, a.nc0, chunk) * sizeof(double) > kResolveSmemMax)
    chunk /= 2;
  a.chunk = chunk;
  const int item_doubles = resolve_item_doubles(a.nx, a.nu, a.nc, a.nc0, chunk);
  const size_t item_bytes = (size_t)item_doubles * sizeof(double);
  if (item_bytes > kResolveSmemMax)
    return cudaErrorInvalidValue;
  int wpc = (int)(kCtaBudget / item_bytes);
  wpc = wpc < 1 ? 1 : (wpc > kMaxWarps ? kMaxWarps : wpc);
  const size_t smem = item_bytes * wpc;
  cudaError_t e = cudaFuncSetAttribute(resolve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess)
    return e;
  const int chunks = (a.nrhs + chunk - 1) / chunk;
  const long items = (long)a.batch * chunks;
  const long grid = (items + wpc - 1) / wpc;
  resolve_kernel<<<(unsigned)grid, wpc * 32, smem, st>>>(a, item_doubles, items, chunks);
  return cudaGetLastError();
}

} // namespace ab2
