// item_launch.cuh -- launch selection shared by the per-item programs (lq_items.cu): resolve, the θ tangent and adjoint,
// and the factorisation's adjoint and tangent.  Items that leave room for others run one per warp, several warps per
// CTA; a factorisation item too large to share an SM runs alone on a CTA of kItemCtaThreads lanes.  Chunked programs
// (resolve, θ) run one warp per (instance, chunk of right-hand sides or directions).
#pragma once
#include <cuda_runtime.h>

namespace ab2 {

constexpr int kItemMaxWarps = 4;          // warps (independent items) per CTA
constexpr int kItemCtaBudget = 96 * 1024; // shared-memory bytes a CTA of warp items aims for; larger items take a CTA
constexpr int kItemCtaThreads = 256;      // lanes of one CTA-wide item
constexpr int kItemSmemMax = 227 * 1024;  // shared memory one CTA may use on sm_90
constexpr int kItemMaxChunk = 32;         // right-hand sides or directions one warp holds on chip

struct ItemWarpCtx {
  int lane, nl;
  __device__ __forceinline__ void sync() const { __syncwarp(); }
};
struct ItemCtaCtx {
  int lane, nl;
  __device__ __forceinline__ void sync() const { __syncthreads(); }
};

// The calling warp's item, item = blockIdx.x * warps + warp index: run(ctx, sm, item) with the warp's item_doubles of
// dynamic shared memory, if item < items.
template <class F> __device__ __forceinline__ void run_warp_item(int item_doubles, long items, F run) {
  extern __shared__ __align__(16) double smem[];
  const int wid = threadIdx.x >> 5;
  const long item = (long)blockIdx.x * (blockDim.x >> 5) + wid;
  if (item >= items)
    return;
  const ItemWarpCtx ctx{(int)(threadIdx.x & 31), 32};
  run(ctx, smem + (size_t)wid * item_doubles, item);
}

// The calling warp's item of a chunked launch, item = b * chunks + c: run(ctx, sm, b, j0, R) on instance b, columns
// [j0, j0 + R) of a.nrhs.  Not built on run_warp_item: nesting the two moves the decode ahead of the shared-memory
// offset and changes the generated code of resolve and θ.
template <class Args, class F>
__device__ __forceinline__ void run_chunk_item(const Args &a, int item_doubles, long items, int chunks, F run) {
  extern __shared__ __align__(16) double smem[];
  const int wid = threadIdx.x >> 5;
  const long item = (long)blockIdx.x * (blockDim.x >> 5) + wid;
  if (item >= items)
    return;
  const long b = item / chunks;
  const int j0 = (int)(item - b * chunks) * a.chunk;
  const int R = a.nrhs - j0 < a.chunk ? a.nrhs - j0 : a.chunk;
  const ItemWarpCtx ctx{(int)(threadIdx.x & 31), 32};
  run(ctx, smem + (size_t)wid * item_doubles, b, j0, R);
}

// warps (items) per CTA of warp items of item_bytes each
inline int item_warps_per_cta(size_t item_bytes) {
  const int wpc = (int)(kItemCtaBudget / item_bytes);
  return wpc < 1 ? 1 : (wpc > kItemMaxWarps ? kItemMaxWarps : wpc);
}

// warp(args, item_doubles): item b = blockIdx.x * warps + warp index; cta(args): item b = blockIdx.x.  One launch;
// cudaErrorInvalidValue when one item does not fit kItemSmemMax.
template <class Args>
cudaError_t launch_items(void (*warp)(const Args, int), void (*cta)(const Args), const Args &a, long batch,
                         size_t item_bytes, cudaStream_t st) {
  if (batch <= 0)
    return cudaSuccess;
  if (item_bytes > kItemSmemMax)
    return cudaErrorInvalidValue;
  cudaError_t e;
  if (item_bytes > kItemCtaBudget) {
    e = cudaFuncSetAttribute(cta, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)item_bytes);
    if (e != cudaSuccess)
      return e;
    cta<<<(unsigned)batch, kItemCtaThreads, item_bytes, st>>>(a);
    return cudaGetLastError();
  }
  const int wpc = item_warps_per_cta(item_bytes);
  const size_t smem = item_bytes * wpc;
  e = cudaFuncSetAttribute(warp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess)
    return e;
  const long grid = (batch + wpc - 1) / wpc;
  warp<<<(unsigned)grid, wpc * 32, smem, st>>>(a, (int)(item_bytes / sizeof(double)));
  return cudaGetLastError();
}

// kernel(args, item_doubles, items, chunks): one warp per (instance, chunk of a.nrhs columns), items = a.batch * chunks.
// a.chunk is min(a.nrhs, kItemMaxChunk), halved until an item of bytes(a.chunk) fits kItemSmemMax; one launch, or
// cudaErrorInvalidValue when one column does not fit.
template <class Args, class Bytes>
cudaError_t launch_chunked_items(void (*kernel)(const Args, int, long, int), Args a, Bytes bytes, cudaStream_t st) {
  if (a.nrhs <= 0 || a.batch <= 0)
    return cudaSuccess;
  int chunk = a.nrhs < kItemMaxChunk ? a.nrhs : kItemMaxChunk;
  while (chunk > 1 && bytes(chunk) > kItemSmemMax)
    chunk /= 2;
  a.chunk = chunk;
  const size_t item_bytes = bytes(chunk);
  if (item_bytes > kItemSmemMax)
    return cudaErrorInvalidValue;
  const int wpc = item_warps_per_cta(item_bytes);
  const size_t smem = item_bytes * wpc;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess)
    return e;
  const int chunks = (a.nrhs + chunk - 1) / chunk;
  const long items = (long)a.batch * chunks;
  const long grid = (items + wpc - 1) / wpc;
  kernel<<<(unsigned)grid, wpc * 32, smem, st>>>(a, (int)(item_bytes / sizeof(double)), items, chunks);
  return cudaGetLastError();
}

} // namespace ab2
