// lq_assemble.cu -- the step BEFORE the sweep, batched on the device:
// SolverProxDDP::updateLQSubproblem (solvers/proxddp/solver-proxddp.hxx:734-805) fused with
// computeProjectedJacobians (:25-69).  Turns the derivative buffers of every (instance,
// knot) into the packed stage / terminal records the sweep reads -- one pass over HBM,
// so a device-resident caller never moves the knots over PCIe.
//
// Pure streaming work (HBM-bound): a warp per record, grid-stride over 8 CTAs per SM of 256
// threads; every source block and the destination record are contiguous and walked with
// unit stride, four elements per lane in flight.
#include <cuda_runtime.h>

#include "../../include/aligator_b200/gar.h"
#include "lq_assemble.h"
#include "lq_record.cuh"

namespace ab2 {

// active row of the product constraint set: the normal-cone projection Jacobian keeps it
// (core/constraint-set.hxx:25-37 with computeActiveSet of equality-constraint.hpp:52-55,
// negative-orthant.hpp:30-33, box-constraint.hpp:39-43 expressed as one test on [lo, hi])
__device__ __forceinline__ bool row_active(double z, double lo, double hi) { return z > hi || z < lo; }

// The map "element e of the record -> (source array, offset, what to do with it)" is the same
// for every record, so each CTA builds it once in shared memory; per element the kernel then
// spends one table look-up instead of an eleven-way block decode.
enum : int { SRC_JX, SRC_JU, SRC_SLACK, SRC_LXX, SRC_LXU, SRC_LUU, SRC_LX, SRC_LU, SRC_CJX, SRC_CJU, SRC_LV, SRC_COUNT };
enum : int { F_DIAG = 1, F_HESS = 2, F_H0 = 4, F_ROW = 8, F_CORR = 16, F_ZERO = 32 };

struct StageTables {
  const double *src[SRC_COUNT];
  const double *hess[SRC_COUNT]; // second operand (dynamics Hessians) of Lxx / Lxu / Luu
  int blk[SRC_COUNT];            // doubles per record of each source
};

// A warp per record (grid-stride), lanes stride over the record's elements
// [A | B | f | Q | S | R | q | r | C | D | d | pad], UNR elements per lane in flight:
// unit-stride reads of every source block and unit-stride writes of the record.
// PI: per-instance preg (and mu_inv, when given) arrays (ab2_gar_assemble_v); false = the scalars of `in`
template <bool PI>
__global__ void __launch_bounds__(256, 4)
    lq_assemble_stage_kernel(const ab2_lq_inputs in, const double *__restrict__ preg_b,
                             const double *__restrict__ mu_inv_b, double *__restrict__ stage, long nrec, int N, int nx,
                             int nu, int nc, int srec) {
  extern __shared__ int2 tab[]; // [srec]: x = source | flags << 8 | row << 16, y = offset in the source block
  __shared__ StageTables T;
  const int nxx = nx * nx, nxu = nx * nu, nuu = nu * nu;
  if (threadIdx.x == 0) {
    const double *srcs[SRC_COUNT] = {in.Jx, in.Ju, in.slack, in.Lxx, in.Lxu, in.Luu, in.Lx, in.Lu, in.cJx, in.cJu, in.Lv};
    const int blks[SRC_COUNT] = {nxx, nxu, nx, nxx, nxu, nuu, nx, nu, nc * nx, nc * nu, nc};
    for (int i = 0; i < SRC_COUNT; ++i) {
      T.src[i] = srcs[i] ? srcs[i] : in.Jx;
      T.hess[i] = nullptr;
      T.blk[i] = blks[i];
    }
    T.hess[SRC_LXX] = in.Hxx;
    T.hess[SRC_LXU] = in.Hxu;
    T.hess[SRC_LUU] = in.Huu;
  }
  for (int e = threadIdx.x; e < srec; e += blockDim.x) {
    int r = e, id, fl = 0, row = 0;
    if (r < nxx) { // knot.A = dd.Jx()  (:755)
      id = SRC_JX;
    } else if ((r -= nxx) < nxu) { // knot.B = dd.Ju()
      id = SRC_JU;
    } else if ((r -= nxu) < nx) { // knot.f = dyn_slacks[t+1]
      id = SRC_SLACK;
    } else if ((r -= nx) < nxx) { // knot.Q = Lxx; diag += preg; += Hxx (EXACT, :770-774); += id.Hxx_ at t = 0 (:803-804)
      id = SRC_LXX;
      fl = ((r % (nx + 1) == 0) ? F_DIAG : 0) | (in.Hxx ? F_HESS : 0) | (in.Hxx0 ? F_H0 : 0);
    } else if ((r -= nxx) < nxu) {
      id = SRC_LXU;
      fl = in.Hxu ? F_HESS : 0;
    } else if ((r -= nxu) < nuu) {
      id = SRC_LUU;
      fl = ((r % (nu + 1) == 0) ? F_DIAG : 0) | (in.Huu ? F_HESS : 0);
    } else if ((r -= nuu) < nx) { // q = Lxs[t] + cstr_lx_corr (:764, 782)
      id = SRC_LX;
      fl = nc > 0 ? F_CORR : 0;
    } else if ((r -= nx) < nu) { // r = Lus[t] + cstr_lu_corr (:765, 783)
      id = SRC_LU;
      fl = nc > 0 ? F_CORR : 0;
    } else if ((r -= nu) < nc * nx) { // knot.C = projected Jx: rows of inactive constraints zeroed (:49-50, 778)
      id = SRC_CJX;
      fl = F_ROW;
      row = r % nc;
    } else if ((r -= nc * nx) < nc * nu) {
      id = SRC_CJU;
      fl = F_ROW;
      row = r % nc;
    } else if ((r -= nc * nu) < nc) { // knot.d = Lvs[t]
      id = SRC_LV;
    } else { // pad to even
      id = SRC_JX;
      fl = F_ZERO;
      r = 0;
    }
    tab[e] = make_int2(id | (fl << 8) | (row << 16), r);
  }
  __syncthreads();

  constexpr int UNR = 4;
  const int lane = threadIdx.x & 31;
  const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long nwarps = ((long)gridDim.x * blockDim.x) >> 5;
  for (long rec = warp; rec < nrec; rec += nwarps) {
    const int t = (int)(rec % N);
    const long inst = rec / N;
    double *dst = stage + rec * srec;
    for (int e0 = 0; e0 < srec; e0 += 32 * UNR) {
      double v[UNR], h[UNR];
      int2 ent[UNR];
#pragma unroll
      for (int u = 0; u < UNR; ++u) { // every streaming operand of the pass is requested here
        const int e = e0 + 32 * u + lane;
        ent[u] = tab[e < srec ? e : 0];
        const int id = ent[u].x & 0xff;
        const long o = rec * T.blk[id] + ent[u].y;
        v[u] = T.src[id][o];
        h[u] = (ent[u].x & (F_HESS << 8)) ? T.hess[id][o] : 0.0;
      }
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        const int id = ent[u].x & 0xff, fl = (ent[u].x >> 8) & 0xff;
        if (fl == 0)
          continue;
        if (fl & F_ZERO)
          v[u] = 0.0;
        if (fl & F_DIAG)
          v[u] += PI ? preg_b[inst] : in.preg;
        if (fl & F_HESS)
          v[u] += h[u];
        if ((fl & F_H0) && t == 0)
          v[u] += in.Hxx0[inst * nxx + ent[u].y];
        if (fl & F_ROW) {
          const int i = ent[u].x >> 16;
          v[u] = row_active(in.shifted[rec * nc + i], in.lo[i], in.hi[i]) ? v[u] : 0.0;
        }
        if (fl & F_CORR) {
          // corr = P^T lv - Ptilde^T lv, lv = Lvs * mu_inv: both products over ALL rows, then
          // subtracted (:46-52)
          const double *P = (id == SRC_LX) ? in.cJx + rec * nc * nx : in.cJu + rec * nc * nu;
          const int jj = ent[u].y;
          double full = 0.0, proj = 0.0;
          for (int i = 0; i < nc; ++i) {
            const double lv = in.Lv[rec * nc + i] * (PI && mu_inv_b ? mu_inv_b[inst] : in.mu_inv);
            const double pij = P[i + (long)jj * nc];
            const double a = row_active(in.shifted[rec * nc + i], in.lo[i], in.hi[i]) ? 1.0 : 0.0;
            full += pij * lv;
            proj += (pij * a) * lv;
          }
          v[u] += full - proj;
        }
      }
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        const int e = e0 + 32 * u + lane;
        if (e < srec)
          dst[e] = v[u];
      }
    }
  }
}

// Terminal knot (:785-795), initial condition (:797-800): a warp per instance.
__global__ void __launch_bounds__(256)
    lq_assemble_term_kernel(const ab2_lq_inputs in, const double *__restrict__ preg_b,
                            const double *__restrict__ mu_inv_b, double *__restrict__ term, double *__restrict__ G0,
                            double *__restrict__ g0, int batch, int N, int nx, int nct, int nc0, int trec) {
  const int lane = threadIdx.x & 31;
  const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long nwarps = ((long)gridDim.x * blockDim.x) >> 5;
  const int nxx = nx * nx;
  const TermOffsets to = term_offsets(nx, nct);
  for (long b = warp; b < batch; b += nwarps) {
    double *dst = term + b * trec;
    const double preg = preg_b ? preg_b[b] : in.preg, mu_inv = mu_inv_b ? mu_inv_b[b] : in.mu_inv;
    for (int e = lane; e < nxx; e += 32) // knot.Q = tcd.Lxx_; diag += preg
      dst[to.Q + e] = in.Lxx_N[b * nxx + e] + ((e % (nx + 1) == 0) ? preg : 0.0) +
               ((N == 0 && in.Hxx0) ? in.Hxx0[b * nxx + e] : 0.0); // stages[0] is the terminal knot when N = 0 (:803-804)
    for (int j = lane; j < nx; j += 32) { // knot.q = Lxs[N] + cstr_lx_corr[N]
      double full = 0.0, proj = 0.0;
      for (int i = 0; i < nct; ++i) {
        const double lv = in.Lv_N[b * nct + i] * mu_inv;
        const double pij = in.cJx_N[b * nct * nx + i + (long)j * nct];
        const double a = row_active(in.shifted_N[b * nct + i], in.loN[i], in.hiN[i]) ? 1.0 : 0.0;
        full += pij * lv;
        proj += (pij * a) * lv;
      }
      dst[to.q + j] = in.Lx_N[b * nx + j] + (full - proj);
    }
    for (int e = lane; e < nct * nx; e += 32) {
      const int i = e % nct;
      dst[to.C + e] =
          row_active(in.shifted_N[b * nct + i], in.loN[i], in.hiN[i]) ? in.cJx_N[b * nct * nx + e] : 0.0;
    }
    for (int e = lane; e < nct; e += 32)
      dst[to.d + e] = in.Lv_N[b * nct + e];
    for (int e = lane; e < nc0 * nx; e += 32) // prob.G0 = id.Jx(), prob.g0 = id.value_
      G0[b * nc0 * nx + e] = in.G0[b * nc0 * nx + e];
    for (int e = lane; e < nc0; e += 32)
      g0[b * nc0 + e] = in.g0[b * nc0 + e];
  }
}

cudaError_t launch_lq_assemble(const ab2_lq_inputs &in, const double *preg_b, const double *mu_inv_b, double *stage, double *term, double *G0, double *g0,
                               int batch, int N, int nx, int nu, int nc, int nct, int nc0, int srec, int trec,
                               cudaStream_t st) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long full = (long)sms * 8; // 8 CTAs of 256 threads per SM: 2048 threads, the SM's limit
  if (N > 0) {
    const long nrec = (long)batch * N;
    long grid = (nrec + 7) / 8; // 8 warps per CTA
    if (grid > full)
      grid = full;
    const size_t tab_bytes = (size_t)srec * sizeof(int2);
    auto kern = preg_b ? lq_assemble_stage_kernel<true> : lq_assemble_stage_kernel<false>;
    cudaError_t e0 = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tab_bytes);
    if (e0 != cudaSuccess)
      return e0;
    kern<<<(int)grid, 256, tab_bytes, st>>>(in, preg_b, mu_inv_b, stage, nrec, N, nx, nu, nc, srec);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess)
      return e;
  }
  long grid = ((long)batch + 7) / 8;
  if (grid > full)
    grid = full;
  lq_assemble_term_kernel<<<(int)grid, 256, 0, st>>>(in, preg_b, mu_inv_b, term, G0, g0, batch, N, nx, nct, nc0, trec);
  return cudaGetLastError();
}

} // namespace ab2
