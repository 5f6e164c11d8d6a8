// lq_tangent.cu -- the streaming kernel in front of the tangent sweep of ab2_gar_tangent.
//
// The LQ solve is the solution of one symmetric KKT system K z = -h, and K is affine in the data, so along a data
// tangent (Kdot, hdot) the solution moves by zdot = -K^-1 (Kdot z + hdot): the SAME LQ problem with the vectors
// replaced by rho = Kdot z + hdot, which the sweep kernels solve unchanged.  tangent_rhs_kernel computes rho from the
// tangent records and the primal z, per stage knot t (lambda_{t+1} = lams[t], sym(M) = (M + M^T) / 2):
//   x-row  rho_q = qdot + sym(Qdot) x + Sdot u + Cdot^T v + Adot^T lambda_{t+1}   (+ G0dot^T lambda_0 at t = 0)
//   u-row  rho_r = rdot + Sdot^T x + sym(Rdot) u + Ddot^T v + Bdot^T lambda_{t+1}
//   v-row  rho_d = ddot + Cdot x + Ddot u
//   l-row  rho_f = fdot + Adot x + Bdot u
// and for the terminal knot and the initial condition rho_qN = qdot_N + sym(Qdot_N) x_N + C_Ndot^T v_N,
// rho_dN = ddot_N + C_Ndot x_N, rho_g0 = g0dot + G0dot x_0.  It writes -rho in the cotangent layout, so that
// launch_adjoint_records, which negates its cotangent, builds the tangent problem with vectors +rho (exactly).
//
// Layout: one warp per stage knot, grid-stride over batch * N knots, then one warp per instance for the terminal
// and initial rows.  The knot's vectors and the tangent record, in tiles of at most kTile doubles, are staged in the
// warp's slice of shared memory by cp.async (16-byte copies when the source is 16-byte aligned), so every load of a
// record is coalesced.  The rows of rho belong to the lanes round-robin; each lane sums its rows in a fixed order
// (tile by tile, block by block, element by element), so the result does not depend on timing: no atomics.
#include <cuda_runtime.h>

#include <stdint.h>

#include "lq_tangent.h"

namespace ab2 {

namespace {
constexpr int kWarps = 8;    // warps per CTA
constexpr int kTile = 512;   // doubles of a record staged per warp at a time (a whole C2 stage record)

__device__ __forceinline__ void cp8(double *dst, const double *src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src)
               : "memory");
}
__device__ __forceinline__ void cp16(double *dst, const double *src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src)
               : "memory");
}
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// n doubles from global src to shared dst (dst 16-byte aligned), issued by the lanes of one warp
__device__ __forceinline__ void stage_copy(double *dst, const double *src, int n, int lane) {
  if (((uintptr_t)src & 15) == 0) {
    for (int k = lane; 2 * k + 1 < n; k += 32)
      cp16(dst + 2 * k, src + 2 * k);
    if ((n & 1) && lane == 0)
      cp8(dst + n - 1, src + n - 1);
  } else {
    for (int k = lane; k < n; k += 32)
      cp8(dst + k, src + k);
  }
}
__device__ __forceinline__ void stage_vec(double *dst, const double *src, int n, int lane) {
  for (int k = lane; k < n; k += 32)
    cp8(dst + k, src + k);
}

// Part of row i of M y (col = false) or of M^T y (col = true) that lies in the staged tile, for the m x n block M
// stored column-major at record offset o; the tile holds record elements [e0, e1).
__device__ __forceinline__ double mv(const double *tile, int e0, int e1, int o, int m, int n, int i, bool col,
                                     const double *y) {
  double s = 0.0;
  if (m <= 0 || n <= 0)
    return s;
  if (col) { // column i: elements o + i m + r, r < m
    const int base = o + i * m;
    const int lo = base > e0 ? base : e0, hi = base + m < e1 ? base + m : e1;
    for (int e = lo; e < hi; ++e)
      s = fma(tile[e - e0], y[e - base], s);
  } else { // row i: elements o + i + c m, c < n
    const int base = o + i;
    const int c0 = base >= e0 ? 0 : (e0 - base + m - 1) / m;
    int c1 = e1 > base ? (e1 - base + m - 1) / m : 0;
    c1 = c1 < n ? c1 : n;
    for (int c = c0; c < c1; ++c)
      s = fma(tile[base + c * m - e0], y[c], s);
  }
  return s;
}
// entry i of the vector block at record offset o, if it lies in the tile
__device__ __forceinline__ double ve(const double *tile, int e0, int e1, int o, int i) {
  const int e = o + i;
  return e >= e0 && e < e1 ? tile[e - e0] : 0.0;
}
} // namespace

__global__ void __launch_bounds__(kWarps * 32, 4) tangent_rhs_kernel(const TangentRhsArgs a, int tile_len, int warp_doubles) {
  extern __shared__ __align__(16) double smem[];
  const AdjointDims d = a.d;
  const int nx = d.nx, nu = d.nu, nc = d.nc, nct = d.nct, nc0 = d.nc0, N = d.N;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  double *tile = smem + (size_t)wid * warp_doubles;
  double *vec = tile + tile_len;
  // stage record offsets (gar.h): [A | B | f | Q | S | R | q | r | C | D | d | pad]
  const int oA = 0, oB = nx * nx, of = oB + nx * nu, oQ = of + nx, oS = oQ + nx * nx, oR = oS + nx * nu,
            oq = oR + nu * nu, orr = oq + nx, oC = orr + nu, oD = oC + nc * nx, od = oD + nc * nu;
  const int nrow = 2 * nx + nu + nc;
  const long nS = (long)d.batch * N, items = nS + d.batch;
  const long w0 = (long)blockIdx.x * kWarps + wid, ws = (long)gridDim.x * kWarps;
  for (long it = w0; it < items; it += ws) {
    if (it < nS) { // stage knot (b, t) = record `it`; rows [q (nx) | r (nu) | d (nc) | f (nx)]
      const long b = it / N;
      const int t = (int)(it - b * N);
      double *x = vec, *u = x + nx, *v = u + nu, *l = v + nc, *acc = l + nx;
      stage_vec(x, a.xs + (it + b) * nx, nx, lane);
      stage_vec(u, a.us + it * nu, nu, lane);
      stage_vec(v, a.vs + it * nc, nc, lane);
      stage_vec(l, a.lams + it * nx, nx, lane);
      for (int r = lane; r < nrow; r += 32)
        acc[r] = 0.0;
      if (a.stage) {
        const double *rec = a.stage + it * d.srec;
        for (int e0 = 0; e0 < d.srec; e0 += tile_len) {
          const int e1 = e0 + tile_len < d.srec ? e0 + tile_len : d.srec;
          stage_copy(tile, rec + e0, e1 - e0, lane);
          cp_wait();
          __syncwarp();
          for (int r = lane; r < nrow; r += 32) {
            double s;
            if (r < nx) {
              const int i = r;
              s = ve(tile, e0, e1, oq, i) +
                  0.5 * (mv(tile, e0, e1, oQ, nx, nx, i, false, x) + mv(tile, e0, e1, oQ, nx, nx, i, true, x)) +
                  mv(tile, e0, e1, oS, nx, nu, i, false, u) + mv(tile, e0, e1, oC, nc, nx, i, true, v) +
                  mv(tile, e0, e1, oA, nx, nx, i, true, l);
            } else if (r < nx + nu) {
              const int i = r - nx;
              s = ve(tile, e0, e1, orr, i) + mv(tile, e0, e1, oS, nx, nu, i, true, x) +
                  0.5 * (mv(tile, e0, e1, oR, nu, nu, i, false, u) + mv(tile, e0, e1, oR, nu, nu, i, true, u)) +
                  mv(tile, e0, e1, oD, nc, nu, i, true, v) + mv(tile, e0, e1, oB, nx, nu, i, true, l);
            } else if (r < nx + nu + nc) {
              const int i = r - nx - nu;
              s = ve(tile, e0, e1, od, i) + mv(tile, e0, e1, oC, nc, nx, i, false, x) +
                  mv(tile, e0, e1, oD, nc, nu, i, false, u);
            } else {
              const int i = r - nx - nu - nc;
              s = ve(tile, e0, e1, of, i) + mv(tile, e0, e1, oA, nx, nx, i, false, x) +
                  mv(tile, e0, e1, oB, nx, nu, i, false, u);
            }
            acc[r] += s;
          }
          __syncwarp(); // the tile is overwritten next
        }
      } else {
        cp_wait();
        __syncwarp();
      }
      const long xo = (it + b) * nx;
      for (int r = lane; r < nrow; r += 32) {
        double s = acc[r];
        if (r < nx) {
          if (t == 0 && a.G0) { // + G0dot^T lambda_0, G0dot column-major [nc0][nx]
            const double *G = a.G0 + b * nc0 * nx + (long)r * nc0, *l0 = a.lam0 + b * nc0;
            double g = 0.0;
            for (int k = 0; k < nc0; ++k)
              g = fma(G[k], l0[k], g);
            s += g;
          }
          a.rxs[xo + r] = -s;
        } else if (r < nx + nu) {
          a.rus[it * nu + r - nx] = -s;
        } else if (r < nx + nu + nc) {
          a.rvs[it * nc + r - nx - nu] = -s;
        } else {
          a.rlams[it * nx + r - nx - nu - nc] = -s;
        }
      }
      __syncwarp(); // the vectors are overwritten next
    } else { // instance b: rows [q_N (nx) | d_N (nct) | g0 (nc0)]; terminal record [Q | q | C | d]
      const long b = it - nS, xo = (b * (N + 1) + N) * nx;
      const int trows = nx + nct + nc0, tQ = 0, tq = nx * nx, tC = tq + nx, td = tC + nct * nx;
      double *x = vec, *v = x + nx, *acc = v + nct;
      stage_vec(x, a.xs + xo, nx, lane);
      stage_vec(v, a.vsT + b * nct, nct, lane);
      for (int r = lane; r < trows; r += 32)
        acc[r] = 0.0;
      if (a.term) {
        const double *rec = a.term + b * d.trec;
        for (int e0 = 0; e0 < d.trec; e0 += tile_len) {
          const int e1 = e0 + tile_len < d.trec ? e0 + tile_len : d.trec;
          stage_copy(tile, rec + e0, e1 - e0, lane);
          cp_wait();
          __syncwarp();
          for (int r = lane; r < nx + nct; r += 32) {
            double s;
            if (r < nx) {
              s = ve(tile, e0, e1, tq, r) +
                  0.5 * (mv(tile, e0, e1, tQ, nx, nx, r, false, x) + mv(tile, e0, e1, tQ, nx, nx, r, true, x)) +
                  mv(tile, e0, e1, tC, nct, nx, r, true, v);
            } else {
              const int i = r - nx;
              s = ve(tile, e0, e1, td, i) + mv(tile, e0, e1, tC, nct, nx, i, false, x);
            }
            acc[r] += s;
          }
          __syncwarp();
        }
      } else {
        cp_wait();
        __syncwarp();
      }
      const double *G = a.G0 ? a.G0 + b * nc0 * nx : nullptr, *l0 = a.lam0 + b * nc0, *x0 = a.xs + b * (N + 1) * nx;
      for (int r = lane; r < trows; r += 32) {
        double s = acc[r];
        if (r < nx) {
          if (N == 0 && G) { // x_0 = x_N: + G0dot^T lambda_0
            double g = 0.0;
            for (int k = 0; k < nc0; ++k)
              g = fma(G[(long)r * nc0 + k], l0[k], g);
            s += g;
          }
          a.rxs[xo + r] = -s;
        } else if (r < nx + nct) {
          a.rvsT[b * nct + r - nx] = -s;
        } else { // rho_g0 = g0dot + G0dot x_0
          const int i = r - nx - nct;
          if (a.g0)
            s += a.g0[b * nc0 + i];
          if (G) {
            double g = 0.0;
            for (int c = 0; c < nx; ++c)
              g = fma(G[i + (long)c * nc0], x0[c], g);
            s += g;
          }
          a.rlam0[b * nc0 + i] = -s;
        }
      }
      __syncwarp();
    }
  }
}

cudaError_t launch_tangent_rhs(const TangentRhsArgs &a, cudaStream_t st) {
  const AdjointDims &d = a.d;
  const long items = (long)d.batch * d.N + d.batch;
  if (items <= 0)
    return cudaSuccess;
  const int longest = d.srec > d.trec ? d.srec : d.trec;
  int tile_len = longest < kTile ? longest : kTile;
  tile_len = (tile_len + 1) & ~1; // keeps every warp's slice 16-byte aligned
  if (tile_len < 2)
    tile_len = 2;
  const int srow = 2 * d.nx + d.nu + d.nc;
  const int tvec = d.nx + d.nct, trow = d.nx + d.nct + d.nc0;
  int warp_doubles = tile_len + (srow > tvec ? srow : tvec) + (srow > trow ? srow : trow);
  warp_doubles = (warp_doubles + 1) & ~1;
  const size_t smem = (size_t)warp_doubles * kWarps * sizeof(double);
  cudaError_t e = cudaFuncSetAttribute(tangent_rhs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess)
    return e;
  int dev = 0, sms = 132, per_sm = 1;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, tangent_rhs_kernel, kWarps * 32, smem);
  if (e != cudaSuccess)
    return e;
  long grid = (items + kWarps - 1) / kWarps;
  const long full = (long)sms * (per_sm > 0 ? per_sm : 1);
  if (grid > full)
    grid = full;
  tangent_rhs_kernel<<<(int)grid, kWarps * 32, smem, st>>>(a, tile_len, warp_doubles);
  return cudaGetLastError();
}

} // namespace ab2
