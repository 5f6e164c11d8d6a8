// kkt_error.h -- host interface of the batched KKT-residual kernel (kkt_error.cu).
#pragma once
#include <cuda_runtime.h>

namespace ab2 {
struct KktErrorArgs {
  int batch, N, nx, nu, nc, nct, nc0, srec, trec;
  int stage_head; // ring head of the stage records (O(1) cycleAppend): knot t in slot (t + head) mod N
  double mueq;
  const double *mueq_b;                             // [batch] per-instance mu (device) or null: mueq for all
  const double *stage, *term, *G0, *g0;             // the problem (packed records)
  const double *xs, *us, *vs, *vsT, *lbd0, *lbdas;  // the solution of the last forward pass
  double *out;                                      // [batch][3]: dyn, cstr, dual
};
cudaError_t launch_kkt_error(const KktErrorArgs &a, cudaStream_t st);
}
