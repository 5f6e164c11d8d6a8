// lq_tangent.h -- host interface of the streaming kernel of ab2_gar_tangent (lq_tangent.cu).
#pragma once
#include <cuda_runtime.h>

#include "lq_adjoint.h"

namespace ab2 {
// The right-hand side rho = Kdot z + hdot of the tangent problem, written NEGATED in the cotangent layout of
// ab2_gar_adjoint, so that launch_adjoint_records (which negates the cotangent) builds the tangent problem.
struct TangentRhsArgs {
  AdjointDims d;
  const double *stage, *term, *G0, *g0;              // tangent records in the problem's layouts; NULL = zero
  const double *xs, *us, *vs, *vsT, *lam0, *lams;    // primal z
  double *rxs, *rus, *rvs, *rvsT, *rlam0, *rlams;    // -rho: [batch][N+1][nx], [batch][N][nu], ... like z
};
cudaError_t launch_tangent_rhs(const TangentRhsArgs &a, cudaStream_t st);
} // namespace ab2
