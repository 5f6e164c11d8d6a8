// lq_jacobian.h -- host interface of the two streaming kernels of ab2_gar_adjoint_many / ab2_gar_tangent_many, which
// ab2_gar_adjoint / ab2_gar_tangent run at nrhs = 1 (lq_jacobian.cu), and of their generalised modes
// (ab2_gar_rho_many / ab2_gar_grad_many).  Every per-right-hand-side array is [nrhs][batch][...]: block j * batch + b is
// right-hand side j of instance b.  The primal z is [batch][...] in the solver's output layouts.
#pragma once
#include <cuda_runtime.h>

#include "lq_adjoint.h"

namespace ab2 {
// A vector in the solution's layouts (xs .. lams), [batch][...] when shared by every right-hand side, [nrhs][batch][...]
// when `each` is set.
struct SolVec {
  const double *xs, *us, *vs, *vsT, *lam0, *lams;
  bool each;
};

// Reverse mode: gradient records of right-hand side j from y_j = resolve(zbar_j) = -K^-1 zbar_j and z:
// dh = y, dK = y z^T read out of K's blocks (the symmetric Q and R get the symmetric part).  With neg, every value is
// negated (pad elements stay +0.0): ab2_gar_adjoint passes its adjoint solution w = -y.
// Generalised mode (ext, ab2_gar_grad_many, never with neg): out_j = Gr^(vec)(y_j; z_j) + Gr_K(y2_j; z2_j), where z
// may be per right-hand side (z_each), Gr_K leaves out the vector blocks (written 0) and the second pair is optional
// (y2.xs == NULL: absent).
struct JacobianGradArgs {
  AdjointDims d;
  int nrhs;
  const double *xs, *us, *vs, *vsT, *lam0, *lams;        // primal z
  const double *yxs, *yus, *yvs, *yvsT, *ylam0, *ylams;  // y, in the solution's layouts
  double *stage, *term, *G0, *g0;                        // any may be NULL: not written
  bool neg;
  bool ext = false, vec = true, z_each = false;
  SolVec y2{}, z2{};                                     // y2.each is ignored: y2 is always per right-hand side
};
// Forward mode: the right-hand side rho_j = Kdot_j z + hdot_j of tangent j, in resolve's rhs layouts (q like xs with
// q_N last, r like us, d like vs, dN like vsT, g0 like lam0, f like lams).
// Generalised mode (ext, ab2_gar_rho_many): out_j = rho^(vec)(Pdot_j; z_j) + rho_K(Pdot2_j; z2_j) + e_j, where z may be
// per right-hand side (z_each), rho_K leaves out the tangent's vector blocks, the second term is optional (two) and e
// ([nrhs][batch], in the solution's layouts) is optional (e.xs == NULL: absent).
struct JacobianRhsArgs {
  AdjointDims d;
  int nrhs;
  const double *stage, *term, *G0, *g0;                  // tangent records in the problem's layouts; NULL = zero
  const double *xs, *us, *vs, *vsT, *lam0, *lams;        // primal z
  double *q, *r, *dv, *dN, *g0out, *f;                   // rho
  bool ext = false, vec = true, z_each = false, two = false;
  const double *stage2 = nullptr, *term2 = nullptr, *G02 = nullptr; // second term's tangent records; NULL = zero
  SolVec z2{}, e{};                                      // e.each is ignored: e is always per right-hand side
};
cudaError_t launch_jacobian_grad(const JacobianGradArgs &a, cudaStream_t st);
cudaError_t launch_jacobian_rhs(const JacobianRhsArgs &a, cudaStream_t st);
} // namespace ab2
