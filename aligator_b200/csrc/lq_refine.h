// lq_refine.h -- host interface of the residual kernel of ab2_gar_refine / ab2_gar_refine_many and ab2_gar_kkt_error
// (lq_refine.cu): the residual r = K z + h of a solution estimate z and its infinity norms.  Every per-right-hand-side
// array is [nrhs][batch][...]: block j * batch + b is right-hand side j of instance b.
#pragma once
#include <cuda_runtime.h>

#include "lq_adjoint.h"

namespace ab2 {
struct RefineResidualArgs {
  AdjointDims d;
  int nrhs;
  int stage_head;                                 // ring head of the stage records
  const double *stage, *term, *G0, *g0;           // the current problem
  double mueq;                                    // scalar mu, or
  const double *mueq_b;                           // [batch] per-instance mu (device), NULL = the scalar
  bool own;                                       // h = the problem's own vectors (nrhs = 1); else h below
  const double *hq, *hr, *hd, *hdN, *hg0, *hf;    // h in resolve's rhs layouts; NULL = zero
  const double *xs, *us, *vs, *vsT, *lam0, *lams; // z, in the solution's layouts
  double *q, *r, *dv, *dN, *g0out, *f;            // r in resolve's rhs layouts; all NULL = not written
  double *norms;                                  // norms[(j * batch + b) * nstride + col] = max |r|; NULL = none
  int nstride, col;
};
// families: norms[(j * batch + b) * nstride + col + 0 / 1 / 2] = the maxima of the dynamics (f, g0), constraint
// (d, d_N) and stationarity (q, r, q_N) rows instead of one maximum in column col.  The norms are maxima: the caller
// zeroes them first.
cudaError_t launch_refine_residual(const RefineResidualArgs &a, bool families, cudaStream_t st);
} // namespace ab2
