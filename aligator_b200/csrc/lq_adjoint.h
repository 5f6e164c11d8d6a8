// lq_adjoint.h -- host interface of the records kernel of ab2_gar_adjoint and ab2_gar_tangent (lq_adjoint.cu), and the
// dimensions every streaming kernel of the LQ solve's derivatives takes.
#pragma once
#include <cuda_runtime.h>

namespace ab2 {
struct AdjointDims {
  int batch, N, nx, nu, nc, nct, nc0, srec, trec;
};
// The current problem's matrices with new vectors: minus a cotangent (adjoint), or a right-hand side rho as it is
// (copy; tangent).
struct AdjointRecordArgs {
  AdjointDims d;
  int stage_head;                                    // ring head of the current stage records
  const double *stage, *term;                        // the current problem
  const double *xs, *us, *vs, *vsT, *lam0, *lams;    // cotangent (a NULL field reads as zero) or rho
  double *adj_stage, *adj_term, *adj_g0;             // [batch][N][srec] in knot order, [batch][trec], [batch][nc0]
  bool copy;                                         // the vectors are the fields themselves, not their negation
};
cudaError_t launch_adjoint_records(const AdjointRecordArgs &a, cudaStream_t st);
} // namespace ab2
