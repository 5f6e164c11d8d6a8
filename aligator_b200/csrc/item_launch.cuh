// item_launch.cuh -- launch selection shared by the per-item programs of resolve and the factorisation's derivatives
// (lq_resolve.cu, lq_factor_adjoint.cu, lq_factor_tangent.cu): items that leave room for others run one per warp,
// several warps per CTA; an item too large to share an SM runs alone on a CTA of kItemCtaThreads lanes (not resolve).
#pragma once
#include <cuda_runtime.h>

namespace ab2 {

constexpr int kItemMaxWarps = 4;          // warps (independent items) per CTA
constexpr int kItemCtaBudget = 96 * 1024; // shared-memory bytes a CTA of warp items aims for; larger items take a CTA
constexpr int kItemCtaThreads = 256;      // lanes of one CTA-wide item

struct ItemWarpCtx {
  int lane, nl;
  __device__ __forceinline__ void sync() const { __syncwarp(); }
};
struct ItemCtaCtx {
  int lane, nl;
  __device__ __forceinline__ void sync() const { __syncthreads(); }
};

// warps (items) per CTA of warp items of item_bytes each
inline int item_warps_per_cta(size_t item_bytes) {
  const int wpc = (int)(kItemCtaBudget / item_bytes);
  return wpc < 1 ? 1 : (wpc > kItemMaxWarps ? kItemMaxWarps : wpc);
}

// warp(args, item_doubles): item b = blockIdx.x * warps + warp index; cta(args): item b = blockIdx.x.  One launch.
template <class Args>
cudaError_t launch_items(void (*warp)(const Args, int), void (*cta)(const Args), const Args &a, long batch,
                         size_t item_bytes, cudaStream_t st) {
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

} // namespace ab2
