// linesearch.h -- host interface of the batched line-search consumers (linesearch.cu).
#pragma once
#include <cuda_runtime.h>

namespace ab2 {
struct LineSearchArgs {
  int batch, N, nx, nu, nc, nct, nc0;
  // the step: the solution of the LQ forward pass (dxs, dus, dvs, dlams of solver-proxddp.hxx:610-611)
  const double *dxs, *dus, *dvs, *dvsT, *dlam0, *dlams;
};
// trial = current + alpha * step for x, u, v, v_N, lam_0, lam_{1..N} (vector-space integrate)
struct LinearStepIO {
  const double *xs, *us, *vs, *vsT, *lam0, *lams; // current iterate, laid out like the step
  double *txs, *tus, *tvs, *tvsT, *tlam0, *tlams; // trial iterate (outputs)
};
// alpha_b: [batch] per-instance step lengths (device) replacing alpha, or null
cudaError_t launch_linear_step(const LineSearchArgs &a, const LinearStepIO &io, double alpha, const double *alpha_b,
                               cudaStream_t st);
// out[b] = sum_t Lxs[b][t].dxs[b][t] (t = 0..N) + sum_t Lus[b][t].dus[b][t] (t = 0..N-1)
cudaError_t launch_directional_derivative(const LineSearchArgs &a, const double *Lxs, const double *Lus, double *out,
                                          cudaStream_t st);
// out[b] = cost[b] + 1/2 (mucstr |lam0|^2 + mudyn sum |lam_{t+1}|^2 + mucstr sum |v_t|^2 + mucstr |v_N|^2)
// (mudyn_b, mucstr_b: [batch] per-instance values (device) replacing mudyn / mucstr, or null)
cudaError_t launch_al_value(int batch, int N, int nx, int nc, int nct, int nc0, const double *lam0, const double *lams,
                            const double *vs, const double *vsT, const double *cost, double mudyn, double mucstr,
                            const double *mudyn_b, const double *mucstr_b, double *out, cudaStream_t st);
} // namespace ab2
