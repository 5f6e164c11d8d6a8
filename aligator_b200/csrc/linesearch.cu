// linesearch.cu -- the consumers of the LQ step inside SolverProxDDP's line search, batched over
// the problem instances so that the inner loop stays on the device (SURVEY section 8f rank 2):
//   * tryLinearStep's vector part (solvers/proxddp/solver-proxddp.hxx:111-155): trial_lams, trial_vs =
//     results + alpha * step (math::vectorMultiplyAdd, :121-124) and trial_xs, trial_us by the
//     vector-space integrate x + alpha dx (:139-150; a manifold's integrate belongs to the
//     modelling library and stays with the caller),
//   * ALFunction::directionalDerivative (solvers/proxddp/merit-function.hxx:68-104) and
//     costDirectionalDerivative (:13-31): sum of Lx.dx and Lu.du over the horizon,
//   * the penalty part of ALFunction::evaluate (:33-66).
// Pure streaming / reduction work: grid-stride axpy, one warp per instance for the reductions
// (lanes stride over the instance's contiguous arrays, shuffle tree at the end).
#include <cuda_runtime.h>

#include "linesearch.h"

namespace ab2 {

// PI: per-instance step lengths alpha_b (ab2_gar_linear_step_v); false = the scalar alpha.  The arrays one after the
// other, each a plain grid-stride loop (`trial` may be `current`, as in the refinement's z += delta).
template <bool PI>
__global__ void __launch_bounds__(256)
    linear_step_kernel(const LineSearchArgs a, const LinearStepIO io, const double alpha, const double *__restrict__ alpha_b) {
#pragma unroll 1
  for (int f = 0; f < 6; ++f) {
    long per; // per: elements of one instance in this array
    const double *cur, *stp;
    double *out;
    if (f == 0) {
      cur = io.xs, stp = a.dxs, out = io.txs, per = (long)(a.N + 1) * a.nx;
    } else if (f == 1) {
      cur = io.us, stp = a.dus, out = io.tus, per = (long)a.N * a.nu;
    } else if (f == 2) {
      cur = io.vs, stp = a.dvs, out = io.tvs, per = (long)a.N * a.nc;
    } else if (f == 3) {
      cur = io.vsT, stp = a.dvsT, out = io.tvsT, per = a.nct;
    } else if (f == 4) {
      cur = io.lam0, stp = a.dlam0, out = io.tlam0, per = a.nc0;
    } else {
      cur = io.lams, stp = a.dlams, out = io.tlams, per = (long)a.N * a.nx;
    }
    for (long j = blockIdx.x * (long)blockDim.x + threadIdx.x; j < per * a.batch; j += (long)gridDim.x * blockDim.x) {
      const double al = PI ? alpha_b[j / per] : alpha; // the alpha of the instance that owns the element
      out[j] = cur[j] + al * stp[j]; // results + alpha * step, as vectorMultiplyAdd / integrate write it
    }
  }
}

__device__ __forceinline__ double warp_sum(double v) {
  for (int o = 16; o > 0; o >>= 1)
    v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(256)
    directional_derivative_kernel(const LineSearchArgs a, const double *__restrict__ Lxs, const double *__restrict__ Lus,
                                  double *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long nwarps = ((long)gridDim.x * blockDim.x) >> 5;
  const long nX = (long)(a.N + 1) * a.nx, nU = (long)a.N * a.nu;
  for (long b = warp; b < a.batch; b += nwarps) {
    double s0 = 0.0, s1 = 0.0; // two chains
    const double *lx = Lxs + b * nX, *dx = a.dxs + b * nX;
    for (long i = lane; i < nX; i += 64) {
      s0 += lx[i] * dx[i];
      if (i + 32 < nX)
        s1 += lx[i + 32] * dx[i + 32];
    }
    const double *lu = Lus + b * nU, *du = a.dus + b * nU;
    for (long i = lane; i < nU; i += 64) {
      s0 += lu[i] * du[i];
      if (i + 32 < nU)
        s1 += lu[i + 32] * du[i + 32];
    }
    const double s = warp_sum(s0 + s1);
    if (lane == 0)
      out[b] = s;
  }
}

__global__ void __launch_bounds__(256)
    al_value_kernel(const int batch, const int N, const int nx, const int nc, const int nct, const int nc0,
                    const double *__restrict__ lam0, const double *__restrict__ lams, const double *__restrict__ vs,
                    const double *__restrict__ vsT, const double *__restrict__ cost, const double mudyn_s,
                    const double mucstr_s, const double *__restrict__ mudyn_b, const double *__restrict__ mucstr_b,
                    double *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long nwarps = ((long)gridDim.x * blockDim.x) >> 5;
  for (long b = warp; b < batch; b += nwarps) {
    const double mudyn = mudyn_b ? mudyn_b[b] : mudyn_s, mucstr = mucstr_b ? mucstr_b[b] : mucstr_s;
    double sl0 = 0.0, sl = 0.0, sv = 0.0;
    for (long i = lane; i < nc0; i += 32)
      sl0 += lam0[b * nc0 + i] * lam0[b * nc0 + i];
    for (long i = lane; i < (long)N * nx; i += 32)
      sl += lams[b * N * nx + i] * lams[b * N * nx + i];
    for (long i = lane; i < (long)N * nc; i += 32)
      sv += vs[b * N * nc + i] * vs[b * N * nc + i];
    for (long i = lane; i < nct; i += 32)
      sv += vsT[b * nct + i] * vsT[b * nct + i];
    const double pen = 0.5 * (mucstr * warp_sum(sl0) + mudyn * warp_sum(sl) + mucstr * warp_sum(sv));
    if (lane == 0)
      out[b] = (cost ? cost[b] : 0.0) + pen;
  }
}

static int grid_for(long work_items, int per_cta) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  long g = (work_items + per_cta - 1) / per_cta;
  if (g > (long)sms * 8)
    g = (long)sms * 8;
  return g < 1 ? 1 : (int)g;
}

cudaError_t launch_linear_step(const LineSearchArgs &a, const LinearStepIO &io, double alpha, const double *alpha_b,
                               cudaStream_t st) {
  const long total = (long)a.batch * ((long)(a.N + 1) * a.nx + (long)a.N * (a.nu + a.nc + a.nx) + a.nct + a.nc0);
  if (alpha_b)
    linear_step_kernel<true><<<grid_for(total, 256 * 4), 256, 0, st>>>(a, io, alpha, alpha_b);
  else
    linear_step_kernel<false><<<grid_for(total, 256 * 4), 256, 0, st>>>(a, io, alpha, alpha_b);
  return cudaGetLastError();
}
cudaError_t launch_directional_derivative(const LineSearchArgs &a, const double *Lxs, const double *Lus, double *out,
                                          cudaStream_t st) {
  directional_derivative_kernel<<<grid_for(a.batch, 8), 256, 0, st>>>(a, Lxs, Lus, out);
  return cudaGetLastError();
}
cudaError_t launch_al_value(int batch, int N, int nx, int nc, int nct, int nc0, const double *lam0, const double *lams,
                            const double *vs, const double *vsT, const double *cost, double mudyn, double mucstr,
                            const double *mudyn_b, const double *mucstr_b, double *out, cudaStream_t st) {
  al_value_kernel<<<grid_for(batch, 8), 256, 0, st>>>(batch, N, nx, nc, nct, nc0, lam0, lams, vs, vsT, cost, mudyn,
                                                        mucstr, mudyn_b, mucstr_b, out);
  return cudaGetLastError();
}

} // namespace ab2
