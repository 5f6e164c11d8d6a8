// proxddp_inner.h -- host interface of the batched multiplier / Lagrangian-gradient / criterion kernels
// (proxddp_inner.cu).
#pragma once
#include <cuda_runtime.h>

#include "../../include/aligator_b200/gar.h"

namespace ab2 {
struct InnerDims {
  int batch, N, nx, nu, nc, nct, nc0;
};
// computeMultipliers (solver-proxddp.hxx:220-318); out2 [batch][2] = [prim_infeas, finite];
// mu_b, mu_dyn_b: [batch] per-instance values (device) replacing in.mu / in.mu_dyn, or null
cudaError_t launch_multipliers(const InnerDims &d, const ab2_mult_inputs &in, const double *mu_b, const double *mu_dyn_b,
                               const ab2_mult_outputs &out, double *out2, cudaStream_t st);
// LagrangianDerivatives::compute (core/lagrangian.hpp:29-92) into the non-NULL outputs
cudaError_t launch_lagrangian_gradient(const InnerDims &d, const ab2_lag_inputs &in, const ab2_lag_outputs &out,
                                       cudaStream_t st);
// computeCriterion (solver-proxddp.hxx:703-732); out2 [batch][2] = [inner_criterion, dual_infeas]
cudaError_t launch_criterion(const InnerDims &d, const double *Lxs, const double *Lus, const double *init_value,
                             const double *slack, const double *Lv, const double *Lv_N, double *out2,
                             cudaStream_t st);
} // namespace ab2
