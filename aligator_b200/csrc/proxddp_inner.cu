// proxddp_inner.cu -- the rest of SolverProxDDP's inner iteration around the sweep, batched over the
// problem instances, so that the LQ right-hand side and the line-search gradients are produced on the device:
//   * computeMultipliers (solvers/proxddp/solver-proxddp.hxx:220-318): dynamics slacks, first-order
//     multiplier estimates, shifted constraints, Lvs, primal infeasibility;
//   * LagrangianDerivatives::compute (core/lagrangian.hpp:29-92): Lxs, Lus at any multiplier set;
//   * computeCriterion (solver-proxddp.hxx:703-732): inner criterion and dual infeasibility.
// The multiplier and criterion kernels are streaming work, one warp per instance (lanes stride over the
// instance's contiguous arrays, shuffle reductions at the end), like linesearch.cu.  The gradient is the
// bandwidth-heavy one (it reads every dynamics and constraint Jacobian): a warp per knot, see below.
#include <cuda_runtime.h>

#include "proxddp_inner.h"

namespace ab2 {

constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ double warp_max(double v) {
  for (int o = 16; o > 0; o >>= 1)
    v = fmax(v, __shfl_xor_sync(kFull, v, o));
  return v;
}

// Normal-cone projection of one constraint row (gar.h): an equality row (lo = +inf) keeps z
// (equality-constraint.hpp:37-40); any other row gives z - max(min(z, hi), lo) (box-constraint.hpp:27-37), the
// clamp written with std::min / std::max's comparisons, as Eigen's cwiseMin(hi).cwiseMax(lo) evaluates it.
__device__ __forceinline__ double normal_cone(double z, double lo, double hi) {
  if (lo == __longlong_as_double(0x7ff0000000000000LL))
    return z;
  double c = (hi < z) ? hi : z;
  c = (c < lo) ? lo : c;
  return z - c;
}

// PI: per-instance mu_b / mu_dyn_b (ab2_gar_multipliers_v); false = the scalars of `in`
template <bool PI>
__global__ void __launch_bounds__(256)
    multipliers_kernel(const InnerDims d, const ab2_mult_inputs in, const double *__restrict__ mu_b,
                       const double *__restrict__ mu_dyn_b, const ab2_mult_outputs out, double *__restrict__ out2) {
  const int lane = threadIdx.x & 31;
  const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long nwarps = ((long)gridDim.x * blockDim.x) >> 5;
  const double mu_s = in.mu, mu_dyn_s = in.mu_dyn, mu_inv_s = 1.0 / mu_s; // mu_inv() = 1 / mu()
  const long nD = (long)d.N * d.nx, nV = (long)d.N * d.nc;
  for (long b = warp; b < d.batch; b += nwarps) {
    const double mu = PI ? mu_b[b] : mu_s, mu_dyn = PI ? mu_dyn_b[b] : mu_dyn_s;
    const double mu_inv = PI ? 1.0 / mu : mu_inv_s; // the same quotient, per instance
    double dyn = 0.0, infeas = 0.0; // |fs|_inf, |stage_infeas|_inf
    bool ok = true;
    // initial constraint: fs[0] = value_, lams_plus[0] = lams[0] + fs[0] / mu()   (:244-248)
    for (int i = lane; i < d.nc0; i += 32) {
      const long o = b * d.nc0 + i;
      const double f = in.init_value[o];
      const double lp = in.lam0[o] + f / mu;
      out.lam0_plus[o] = lp;
      ok &= isfinite(lp);
      dyn = fmax(dyn, fabs(f));
    }
    // dynamics: fs[t+1] = xnext_t (-) x_{t+1}, lams_plus[t+1] = lams[t+1] + fs[t+1] / mu_dyn()   (:263-265)
    for (long i = lane; i < nD; i += 32) {
      const long o = b * nD + i;
      const double f = in.fs ? in.fs[o] : in.xnext[o] - in.xs[b * (nD + d.nx) + d.nx + i];
      out.slack[o] = f;
      const double lp = in.lams[o] + f / mu_dyn;
      out.lams_plus[o] = lp;
      ok &= isfinite(lp);
      dyn = fmax(dyn, fabs(f));
    }
    // path constraints   (:271-289)
    for (long i = lane; i < nV; i += 32) {
      const long o = b * nV + i;
      const int row = (int)(i % d.nc);
      const double prev = in.prev_vs[o];
      const double z = in.cval[o] + mu * prev; // shifted_constraints += mu() * vs_prev   (:277)
      out.shifted[o] = z;
      const double n = normal_cone(z, in.lo[row], in.hi[row]); // (:278)
      const double lv = n - mu * in.vs[o];                      // Lvs = vs_plus - mu() * vs   (:281-282)
      const double vp = mu_inv * n;                             // vs_plus = mu_inv() * vs_plus   (:283)
      out.Lv[o] = lv;
      out.vs_plus[o] = vp;
      infeas = fmax(infeas, fabs(mu * (vp - prev))); // stage_infeas = mu() * (vs_plus - vs_prev)   (:286)
      ok &= isfinite(lv);
    }
    // terminal constraints, only when there are any   (:292-314)
    for (int i = lane; i < d.nct; i += 32) {
      const long o = b * d.nct + i;
      const double prev = in.prev_vsT[o];
      const double z = in.cval_N[o] + mu * prev;
      out.shifted_N[o] = z;
      const double n = normal_cone(z, in.loN[i], in.hiN[i]);
      const double lv = n - mu * in.vsT[o];
      const double vp = mu_inv * n;
      out.Lv_N[o] = lv;
      out.vsT_plus[o] = vp;
      infeas = fmax(infeas, fabs(mu * (vp - prev)));
      ok &= isfinite(lv);
    }
    const double prim = fmax(warp_max(infeas), warp_max(dyn)); // (:315-316)
    const bool all_ok = __all_sync(kFull, ok);
    if (lane == 0) {
      out2[2 * b] = prim;
      out2[2 * b + 1] = all_ok ? 1.0 : 0.0;
    }
  }
}

// Lagrangian gradient.  A warp per knot (instance b, knot t = 0..N).  Every output entry is one column of the
// knot's Jacobians dotted with the multipliers:
//     column c of [Jx | Ju] . lam_{t+1}  +  column c of [cJx | cJu] . v_t  (+ column c of G0 . lam0 at t = 0)
// (terminal knot: cJx_N . v_N, plus G0 . lam0 when N = 0).  The Jacobians are column-major, so columns
// c0 .. c0 + w - 1 of a block are one contiguous run of doubles (two when the run crosses from the x block into the
// u block).  The warp copies these runs into its shared-memory tile with unit-stride loads -- independent of each
// other, so every lane keeps several in flight -- and then lane c sums column c0 + c out of the tile.  Each lane
// starts at row c mod rows, which spreads the lanes' tile addresses over the banks.  A chunk has w <= 32 columns,
// as many as the tile holds.
__device__ __forceinline__ double split_load(const double *xb, const double *ub, long xsize, long g) {
  return g < xsize ? xb[g] : ub[g - xsize];
}
__device__ __forceinline__ double col_dot(const double *col, const double *y, int rows, int start) {
  double acc = 0.0;
  int i = start;
  for (int j = 0; j < rows; ++j) {
    acc += col[i] * y[i];
    if (++i == rows)
      i = 0;
  }
  return acc;
}

__global__ void __launch_bounds__(256)
    lagrangian_gradient_kernel(const InnerDims d, const ab2_lag_inputs in, const ab2_lag_outputs out, const int tile_doubles,
                               const int wmax) {
  extern __shared__ double smem[];
  const int lane = threadIdx.x & 31;
  const int ymax = d.nx + (d.nc > d.nct ? d.nc : d.nct) + d.nc0;
  double *tile = smem + (size_t)(threadIdx.x >> 5) * (tile_doubles + ymax); // this warp's tile, then its multipliers
  double *ys = tile + tile_doubles;
  const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long nwarps = ((long)gridDim.x * blockDim.x) >> 5;
  const int N = d.N, nx = d.nx, nu = d.nu;
  const long nrec = (long)d.batch * (N + 1);
  for (long k = warp; k < nrec; k += nwarps) {
    const long b = k / (N + 1);
    const int t = (int)(k - b * (N + 1));
    const bool term = (t == N);
    const long kn = b * N + t; // stage knot index (t < N)
    const int ncols = term ? nx : nx + nu;
    // dynamics block [Jx | Ju] (nx rows) . lam_{t+1}   (lagrangian.hpp:63-64)
    const int r1 = term ? 0 : nx;
    const double *J1x = term ? nullptr : in.Jx + kn * nx * nx, *J1u = term ? nullptr : in.Ju + kn * nx * nu;
    const double *y1 = term ? nullptr : in.lams + kn * nx;
    // constraint block [cJx | cJu] (nc rows) . v_t, terminal cJx_N (nct rows) . v_N   (:67-72, :85-90)
    const int r2 = term ? d.nct : d.nc;
    const double *J2x = term ? in.cJx_N + b * d.nct * nx : in.cJx + kn * d.nc * nx;
    const double *J2u = term ? nullptr : in.cJu + kn * d.nc * nu;
    const double *y2 = term ? in.vsT + b * d.nct : in.vs + kn * d.nc;
    // initial condition G0 (nc0 rows) . lam0, state columns of knot 0 only   (:51-53)
    const int r3 = (t == 0) ? d.nc0 : 0;
    const double *J3 = in.G0 + b * d.nc0 * nx, *y3 = in.lam0 + b * d.nc0;
    double *y1s = ys, *y2s = ys + r1, *y3s = ys + r1 + r2;
    __syncwarp(); // the previous knot's last chunk has been read
    for (int i = lane; i < r1; i += 32)
      y1s[i] = y1[i];
    for (int i = lane; i < r2; i += 32)
      y2s[i] = y2[i];
    for (int i = lane; i < r3; i += 32)
      y3s[i] = y3[i];
    for (int c0 = 0; c0 < ncols; c0 += wmax) {
      const int w = min(wmax, ncols - c0);
      const int w3 = c0 < nx ? min(w, nx - c0) : 0; // G0 has state columns only
      const int n1 = w * r1, n2 = w * r2, n3 = w3 * r3;
      double *t1 = tile, *t2 = tile + n1, *t3 = tile + n1 + n2;
      __syncwarp(); // the previous chunk has been read
#pragma unroll 4
      for (int e = lane; e < n1; e += 32)
        t1[e] = split_load(J1x, J1u, (long)nx * r1, (long)c0 * r1 + e);
#pragma unroll 4
      for (int e = lane; e < n2; e += 32)
        t2[e] = split_load(J2x, J2u, (long)nx * r2, (long)c0 * r2 + e);
      for (int e = lane; e < n3; e += 32)
        t3[e] = J3[(long)c0 * r3 + e];
      // this lane's cost-gradient entry, requested before the tile is read
      const int c = c0 + lane;
      double g = 0.0;
      if (lane < w) {
        if (c < nx) { // Lxs[t] = -lams[t] (t >= 1, set by the previous stage, :74-76) + cost Lx_ (:60, :84)
          g = term ? in.lx_N[b * nx + c] : in.lx[kn * nx + c];
          if (t >= 1)
            g = -in.lams[(b * N + t - 1) * nx + c] + g;
        } else { // Lus[t] = cost Lu_ (:61)
          g = in.lu[kn * nu + (c - nx)];
        }
      }
      __syncwarp();
      if (lane >= w)
        continue;
      double acc = r1 ? col_dot(t1 + lane * r1, y1s, r1, lane % r1) : 0.0;
      if (r2)
        acc += col_dot(t2 + lane * r2, y2s, r2, lane % r2);
      if (lane < w3 && r3)
        acc += col_dot(t3 + lane * r3, y3s, r3, lane % r3);
      double v = g + acc;
      if (c < nx) {
        if (t == 0 && in.force_initial_condition) // innerLoop: Lxs[0].setZero()   (solver-proxddp.hxx:592-594)
          v = 0.0;
        if (term) {
          if (out.Lx_N)
            out.Lx_N[b * nx + c] = v;
        } else if (out.Lx) {
          out.Lx[kn * nx + c] = v;
        }
        if (out.Lxs)
          out.Lxs[k * nx + c] = v;
      } else {
        const long o = kn * nu + (c - nx);
        if (out.Lu)
          out.Lu[o] = v;
        if (out.Lus)
          out.Lus[o] = v;
      }
    }
  }
}

__global__ void __launch_bounds__(256)
    criterion_kernel(const InnerDims d, const double *__restrict__ Lxs, const double *__restrict__ Lus,
                     const double *__restrict__ init_value, const double *__restrict__ slack, const double *__restrict__ Lv,
                     const double *__restrict__ Lv_N, double *__restrict__ out2) {
  const int lane = threadIdx.x & 31;
  const long warp = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long nwarps = ((long)gridDim.x * blockDim.x) >> 5;
  const long nX = (long)(d.N + 1) * d.nx, nU = (long)d.N * d.nu, nV = (long)d.N * d.nc;
  // stage i's dynamics residual is dyn_slacks[i] (:715): fs0 and fs_1..fs_{N-1} = slack knots 0..N-2
  const long nS = d.N >= 1 ? (long)(d.N - 1) * d.nx : 0;
  const int n0 = d.N >= 1 ? d.nc0 : 0;
  for (long b = warp; b < d.batch; b += nwarps) {
    double dual = 0.0, other = 0.0;
    for (long i = lane; i < nX; i += 32) // rx over knots 0..N   (:712, :723)
      dual = fmax(dual, fabs(Lxs[b * nX + i]));
    for (long i = lane; i < nU; i += 32) // ru   (:713)
      dual = fmax(dual, fabs(Lus[b * nU + i]));
    for (int i = lane; i < n0; i += 32) // rd of stage 0   (:715)
      other = fmax(other, fabs(init_value[b * d.nc0 + i]));
    for (long i = lane; i < nS; i += 32) // rd of stages 1..N-1
      other = fmax(other, fabs(slack[b * (long)d.N * d.nx + i]));
    for (long i = lane; i < nV; i += 32) // rc   (:717)
      other = fmax(other, fabs(Lv[b * nV + i]));
    for (int i = lane; i < d.nct; i += 32) // rc of the terminal knot   (:724)
      other = fmax(other, fabs(Lv_N[b * d.nct + i]));
    dual = warp_max(dual);
    other = warp_max(other);
    if (lane == 0) {
      out2[2 * b] = fmax(dual, other); // inner_criterion   (:728)
      out2[2 * b + 1] = dual;          // dual_infeas   (:729-731)
    }
  }
}

static int sm_count() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

static int warp_grid(long warps_needed) { // 8 warps per CTA, at most 8 CTAs per SM
  long g = (warps_needed + 7) / 8;
  const long cap = (long)sm_count() * 8;
  if (g > cap)
    g = cap;
  return g < 1 ? 1 : (int)g;
}

cudaError_t launch_multipliers(const InnerDims &d, const ab2_mult_inputs &in, const double *mu_b, const double *mu_dyn_b,
                               const ab2_mult_outputs &out, double *out2, cudaStream_t st) {
  if (mu_b)
    multipliers_kernel<true><<<warp_grid(d.batch), 256, 0, st>>>(d, in, mu_b, mu_dyn_b, out, out2);
  else
    multipliers_kernel<false><<<warp_grid(d.batch), 256, 0, st>>>(d, in, mu_b, mu_dyn_b, out, out2);
  return cudaGetLastError();
}

cudaError_t launch_lagrangian_gradient(const InnerDims &d, const ab2_lag_inputs &in, const ab2_lag_outputs &out,
                                       cudaStream_t st) {
  // rows of one tile column: the dynamics, constraint and initial-condition blocks stacked
  const int rows = (d.N > 0 ? d.nx : 0) + (d.nc > d.nct ? d.nc : d.nct) + d.nc0;
  const int tile = rows > 1024 ? rows : 1024; // 8 KB per warp
  int wmax = tile / (rows > 0 ? rows : 1);
  wmax = wmax > 32 ? 32 : wmax;
  const int ymax = d.nx + (d.nc > d.nct ? d.nc : d.nct) + d.nc0;
  const size_t smem = (size_t)8 * (tile + ymax) * sizeof(double); // 8 warps per CTA
  cudaError_t e = cudaFuncSetAttribute(lagrangian_gradient_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess)
    return e;
  int per_sm = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lagrangian_gradient_kernel, 256, smem);
  if (e != cudaSuccess)
    return e;
  const long nrec = (long)d.batch * (d.N + 1);
  long grid = (nrec + 7) / 8;
  const long cap = (long)sm_count() * (per_sm > 0 ? per_sm : 1);
  if (grid > cap)
    grid = cap;
  lagrangian_gradient_kernel<<<(int)grid, 256, smem, st>>>(d, in, out, tile, wmax);
  return cudaGetLastError();
}

cudaError_t launch_criterion(const InnerDims &d, const double *Lxs, const double *Lus, const double *init_value,
                             const double *slack, const double *Lv, const double *Lv_N, double *out2,
                             cudaStream_t st) {
  criterion_kernel<<<warp_grid(d.batch), 256, 0, st>>>(d, Lxs, Lus, init_value, slack, Lv, Lv_N, out2);
  return cudaGetLastError();
}

} // namespace ab2
