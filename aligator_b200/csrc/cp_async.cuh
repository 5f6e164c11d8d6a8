// cp_async.cuh -- staging of global memory in shared memory by cp.async, issued by the lanes of one warp
// (lq_jacobian.cu, lq_refine.cu).
#pragma once
#include <cuda_runtime.h>

#include <stdint.h>

namespace ab2 {

__device__ __forceinline__ void cp8(double *dst, const double *src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src)
               : "memory");
}
__device__ __forceinline__ void cp16(double *dst, const double *src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src)
               : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_wait_prev() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }
__device__ __forceinline__ void cp_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// n doubles from global src to shared dst (dst 16-byte aligned), issued by the lanes of one warp
__device__ __forceinline__ void stage_copy(double *dst, const double *src, int n, int lane) {
  if (((uintptr_t)src & 15) == 0) {
    for (int k = lane; 2 * k + 1 < n; k += 32)
      cp16(dst + 2 * k, src + 2 * k);
    if ((n & 1) && lane == 0)
      cp8(dst + n - 1, src + n - 1);
  } else {
    for (int k = lane; k < n; k += 32)
      cp8(dst + k, src + k);
  }
}

} // namespace ab2
