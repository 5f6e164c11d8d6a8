// lq_items.h -- host interface of the per-item kernels (lq_items.cu): ab2_gar_resolve (program in lq_resolve.cuh),
// ab2_gar_theta_tangent and ab2_gar_theta_adjoint (lq_theta.cuh), ab2_gar_factor_adjoint (lq_factor_adjoint.cuh) and
// ab2_gar_factor_tangent (lq_factor_tangent.cuh).  Each returns cudaErrorInvalidValue when one column (resolve, θ) or
// one instance (factorisation) does not fit kItemSmemMax; the C ABI refuses such a shape before launching.
#pragma once
#include <cuda_runtime.h>

#include "item_launch.cuh"
#include "lq_factor_adjoint.cuh"
#include "lq_factor_tangent.cuh"
#include "lq_resolve.cuh"
#include "lq_theta.cuh"

namespace ab2 {
// One warp per (instance, chunk of right-hand sides or directions); a.chunk is chosen here.
cudaError_t launch_resolve(ResolveArgs a, cudaStream_t st);
cudaError_t launch_theta_tangent(ThetaArgs a, cudaStream_t st);
cudaError_t launch_theta_adjoint(ThetaArgs a, cudaStream_t st);
// One warp per instance, or one CTA per instance when an item is too large for several to share an SM.
cudaError_t launch_factor_adjoint(const FactorAdjointArgs &a, cudaStream_t st);
cudaError_t launch_factor_tangent(const FactorTangentArgs &a, cudaStream_t st);
} // namespace ab2
