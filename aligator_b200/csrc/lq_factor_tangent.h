// lq_factor_tangent.h -- host interface of the kernel of ab2_gar_factor_tangent (lq_factor_tangent.cu, program in
// lq_factor_tangent.cuh).
#pragma once
#include <cuda_runtime.h>

#include "lq_factor_tangent.cuh"

namespace ab2 {
constexpr int kFactorTangentSmemMax = 227 * 1024; // shared memory one CTA may use on sm_90
// One warp per instance, or one CTA per instance when an item is too large for several to share an SM.
cudaError_t launch_factor_tangent(const FactorTangentArgs &a, cudaStream_t st);
} // namespace ab2
