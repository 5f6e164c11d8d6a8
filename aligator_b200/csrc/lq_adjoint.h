// lq_adjoint.h -- host interface of the two streaming kernels of ab2_gar_adjoint (lq_adjoint.cu).
#pragma once
#include <cuda_runtime.h>

namespace ab2 {
struct AdjointDims {
  int batch, N, nx, nu, nc, nct, nc0, srec, trec;
};
// Step 1: the adjoint problem -- the current problem's matrices with the cotangent-derived vectors.
struct AdjointRecordArgs {
  AdjointDims d;
  int stage_head;                                    // ring head of the current stage records
  const double *stage, *term;                        // the current problem
  const double *xs, *us, *vs, *vsT, *lam0, *lams;    // cotangent; a NULL field reads as zero
  double *adj_stage, *adj_term, *adj_g0;             // [batch][N][srec] in knot order, [batch][trec], [batch][nc0]
};
// Step 3: gradient records from the primal solution z and the adjoint solution w.
struct AdjointGradArgs {
  AdjointDims d;
  const double *xs, *us, *vs, *vsT, *lam0, *lams;        // primal z
  const double *wxs, *wus, *wvs, *wvsT, *wlam0, *wlams;  // adjoint w (the handle's trajectory outputs)
  double *stage, *term, *G0, *g0;                        // any may be NULL: not written
};
cudaError_t launch_adjoint_records(const AdjointRecordArgs &a, cudaStream_t st);
cudaError_t launch_adjoint_grad(const AdjointGradArgs &a, cudaStream_t st);
} // namespace ab2
