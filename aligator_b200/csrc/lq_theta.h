// lq_theta.h -- host interface of the kernels of ab2_gar_theta_tangent and ab2_gar_theta_adjoint (lq_theta.cu,
// programs in lq_theta.cuh).
#pragma once
#include <cuda_runtime.h>

#include "lq_theta.cuh"

namespace ab2 {
constexpr int kThetaSmemMax = 227 * 1024; // shared memory one CTA may use on sm_90
// One warp per (instance, chunk of directions); a.chunk is chosen here.  cudaErrorInvalidValue when one direction
// does not fit kThetaSmemMax (the C ABI refuses such a shape before launching).
cudaError_t launch_theta_tangent(ThetaArgs a, cudaStream_t st);
cudaError_t launch_theta_adjoint(ThetaArgs a, cudaStream_t st);
} // namespace ab2
