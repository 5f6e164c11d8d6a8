// lq_jacobian.h -- host interface of the two streaming kernels of ab2_gar_adjoint_many / ab2_gar_tangent_many, which
// ab2_gar_adjoint / ab2_gar_tangent run at nrhs = 1 (lq_jacobian.cu).  Every per-right-hand-side array is [nrhs][batch][...]: block j * batch + b is right-hand side j of
// instance b.  The primal z is [batch][...] in the solver's output layouts.
#pragma once
#include <cuda_runtime.h>

#include "lq_adjoint.h"

namespace ab2 {
// Reverse mode: gradient records of right-hand side j from y_j = resolve(zbar_j) = -K^-1 zbar_j and z:
// dh = y, dK = y z^T read out of K's blocks (the symmetric Q and R get the symmetric part).  With neg, every value is
// negated (pad elements stay +0.0): ab2_gar_adjoint passes its adjoint solution w = -y.
struct JacobianGradArgs {
  AdjointDims d;
  int nrhs;
  const double *xs, *us, *vs, *vsT, *lam0, *lams;        // primal z
  const double *yxs, *yus, *yvs, *yvsT, *ylam0, *ylams;  // y, in the solution's layouts
  double *stage, *term, *G0, *g0;                        // any may be NULL: not written
  bool neg;
};
// Forward mode: the right-hand side rho_j = Kdot_j z + hdot_j of tangent j, in resolve's rhs layouts (q like xs with
// q_N last, r like us, d like vs, dN like vsT, g0 like lam0, f like lams).
struct JacobianRhsArgs {
  AdjointDims d;
  int nrhs;
  const double *stage, *term, *G0, *g0;                  // tangent records in the problem's layouts; NULL = zero
  const double *xs, *us, *vs, *vsT, *lam0, *lams;        // primal z
  double *q, *r, *dv, *dN, *g0out, *f;                   // rho
};
cudaError_t launch_jacobian_grad(const JacobianGradArgs &a, cudaStream_t st);
cudaError_t launch_jacobian_rhs(const JacobianRhsArgs &a, cudaStream_t st);
} // namespace ab2
