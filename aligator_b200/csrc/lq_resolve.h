// lq_resolve.h -- host interface of the kernel of ab2_gar_resolve (lq_resolve.cu, program in lq_resolve.cuh).
#pragma once
#include <cuda_runtime.h>

#include "lq_resolve.cuh"

namespace ab2 {
constexpr int kResolveSmemMax = 227 * 1024; // shared memory one CTA may use on sm_90
// One warp per (instance, chunk of right-hand sides); a.chunk is chosen here.
cudaError_t launch_resolve(ResolveArgs a, cudaStream_t st);
} // namespace ab2
