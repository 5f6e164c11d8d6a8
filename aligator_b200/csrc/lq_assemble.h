// lq_assemble.h -- host interface of the batched LQ assembly (lq_assemble.cu).
#pragma once
#include <cuda_runtime.h>

#include "../../include/aligator_b200/gar.h"

namespace ab2 {
// preg_b, mu_inv_b: [batch] per-instance values (device) replacing in.preg / in.mu_inv, or null
cudaError_t launch_lq_assemble(const ab2_lq_inputs &in, const double *preg_b, const double *mu_inv_b, double *stage, double *term, double *G0, double *g0,
                               int batch, int N, int nx, int nu, int nc, int nct, int nc0, int srec, int trec,
                               cudaStream_t st);
}
