// kkt_error.cu -- lqrComputeKktError (gar/utils.hxx:88-182) for every instance of the batch, on the
// device: the infinity norms of the dynamics, constraint and stationarity residuals of the
// solution the sweep just produced.  One warp per (instance, knot): lane = residual row (lanes
// walk the columns of the column-major blocks with unit stride), the per-instance maxima meet
// through atomicMax on the bit patterns (non-negative doubles order like unsigned integers, and
// a NaN sorts above every number: it survives).
// Lets a caller -- and the tests -- check ALL instances of a full-size batch without a CPU solver.
#include <cuda_runtime.h>

#include "kkt_error.h"
#include "lq_record.cuh"

namespace ab2 {

__device__ __forceinline__ void atomic_max_nonneg(double *addr, double v) {
  atomicMax(reinterpret_cast<unsigned long long *>(addr), (unsigned long long)__double_as_longlong(v));
}

// running infinity norm that keeps a NaN once it has seen one (fmax would drop it: a residual
// that is not a number must not read as "converged")
__device__ __forceinline__ double upd(double m, double s) {
  const double v = fabs(s);
  return (v > m || v != v) ? v : m;
}

__global__ void __launch_bounds__(256) kkt_error_kernel(const KktErrorArgs a) {
  const int lane = threadIdx.x & 31;
  const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long nwarps = ((long)gridDim.x * blockDim.x) >> 5;
  const int N = a.N, nx = a.nx, nu = a.nu, nc = a.nc, nct = a.nct, nc0 = a.nc0;
  const int nxx = nx * nx, nxu = nx * nu;
  for (long w = warp; w < (long)a.batch * (N + 1); w += nwarps) {
    const long b = w / (N + 1);
    const int t = (int)(w % (N + 1));
    const bool term = t == N;
    const double *x = a.xs + (b * (N + 1) + t) * nx;
    const double *u = term ? nullptr : a.us + (b * N + t) * nu;
    const int ncc = term ? nct : nc, nuu = term ? 0 : nu;
    const double *v = term ? a.vsT + b * nct : a.vs + (b * N + t) * nc;
    const int slot = term ? 0 : ring_slot(t, a.stage_head, N);
    const double *rec = term ? a.term + b * a.trec : a.stage + (b * N + slot) * a.srec;
    // block pointers inside the record
    const double *A = rec, *B = rec + nxx, *f = B + nxu;
    const double *Q = term ? rec : f + nx, *S = Q + nxx, *R = S + nxu;
    const double *q = term ? rec + nxx : R + nu * nu, *r = q + nx;
    const double *C = term ? q + nx : r + nu, *D = C + nc * nx, *d = term ? C + nct * nx : D + nc * nu;
    const double *lam = (t == 0) ? a.lbd0 + b * nc0 : a.lbdas + (b * N + (t - 1)) * nx;
    const double *lamn = term ? nullptr : a.lbdas + (b * N + t) * nx; // lbda_{t+1}
    const double *xn = term ? nullptr : a.xs + (b * (N + 1) + t + 1) * nx;
    double dynE = 0.0, cstE = 0.0, dualE = 0.0;
    if (t == 0) // initial condition G0 x0 + g0 (:96-99)
      for (int i = lane; i < nc0; i += 32) {
        double s = a.g0[b * nc0 + i];
        for (int c = 0; c < nx; ++c)
          s += a.G0[b * nc0 * nx + i + (long)c * nc0] * x[c];
        dynE = upd(dynE, s);
      }
    for (int i = lane; i < ncc; i += 32) { // C x + D u + d - mu v (:110-116)
      double s = d[i] - (a.mueq_b ? a.mueq_b[b] : a.mueq) * v[i];
      for (int c = 0; c < nx; ++c)
        s += C[i + (long)c * ncc] * x[c];
      for (int c = 0; c < nuu; ++c)
        s += D[i + (long)c * ncc] * u[c];
      cstE = upd(cstE, s);
    }
    for (int i = lane; i < nx; i += 32) { // gx (:118-146)
      double s = q[i];
      for (int c = 0; c < nx; ++c)
        s += Q[i + (long)c * nx] * x[c];
      for (int c = 0; c < ncc; ++c)
        s += C[c + (long)i * ncc] * v[c];
      for (int c = 0; c < nuu; ++c)
        s += S[i + (long)c * nx] * u[c];
      if (t == 0) {
        for (int c = 0; c < nc0; ++c)
          s += a.G0[b * nc0 * nx + c + (long)i * nc0] * lam[c];
      } else {
        s -= lam[i];
      }
      if (!term)
        for (int c = 0; c < nx; ++c)
          s += A[c + (long)i * nx] * lamn[c];
      dualE = upd(dualE, s);
    }
    for (int i = lane; i < nuu; i += 32) { // gu
      double s = r[i];
      for (int c = 0; c < nx; ++c)
        s += S[c + (long)i * nx] * x[c];
      for (int c = 0; c < ncc; ++c)
        s += D[c + (long)i * ncc] * v[c];
      for (int c = 0; c < nu; ++c)
        s += R[i + (long)c * nu] * u[c];
      for (int c = 0; c < nx; ++c)
        s += B[c + (long)i * nx] * lamn[c];
      dualE = upd(dualE, s);
    }
    if (!term)
      for (int i = lane; i < nx; i += 32) { // A x + B u + f - x+  (:148-151)
        double s = f[i] - xn[i];
        for (int c = 0; c < nx; ++c)
          s += A[i + (long)c * nx] * x[c];
        for (int c = 0; c < nu; ++c)
          s += B[i + (long)c * nx] * u[c];
        dynE = upd(dynE, s);
      }
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) {
      dynE = upd(dynE, __shfl_xor_sync(0xffffffffu, dynE, m));
      cstE = upd(cstE, __shfl_xor_sync(0xffffffffu, cstE, m));
      dualE = upd(dualE, __shfl_xor_sync(0xffffffffu, dualE, m));
    }
    if (lane == 0) {
      atomic_max_nonneg(a.out + b * 3 + 0, dynE);
      atomic_max_nonneg(a.out + b * 3 + 1, cstE);
      atomic_max_nonneg(a.out + b * 3 + 2, dualE);
    }
  }
}

cudaError_t launch_kkt_error(const KktErrorArgs &a, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(a.out, 0, (size_t)a.batch * 3 * sizeof(double), st);
  if (e != cudaSuccess)
    return e;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  long work = (long)a.batch * (a.N + 1);
  long grid = (work + 7) / 8;
  if (grid > (long)sms * 8)
    grid = (long)sms * 8;
  kkt_error_kernel<<<(int)grid, 256, 0, st>>>(a);
  return cudaGetLastError();
}

} // namespace ab2
