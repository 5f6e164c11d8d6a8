// lq_jacobian.cu -- the two streaming kernels of ab2_gar_adjoint_many and ab2_gar_tangent_many: many cotangents or
// tangents per factorisation, around ab2_gar_resolve's program (lq_resolve.cuh), which solves z = resolve(h) = -K^-1 h.
// ab2_gar_adjoint and ab2_gar_tangent run the same kernels at nrhs = 1 around their own sweep (gar_cuda.cu).
//  * jacobian_grad_kernel: reverse mode.  For cotangent j, y_j = resolve(zbar_j) = -K^-1 zbar_j, so the gradients of
//    ab2_gar_adjoint (dh = -w, dK = -w z^T with w = K^-1 zbar) are dh = y_j and dK = y_j z^T read out of K's blocks:
//      dA = y_l x^T + l y_x^T, dQ = 1/2 (y_x x^T + x y_x^T), dq = y_x, ...   (gar.h, ab2_gar_adjoint)
//    Every element is one or two products, computed by one lane: no sums, no atomics.  ab2_gar_adjoint passes its
//    own w as y and asks for the values negated.
//  * jacobian_rhs_kernel: forward mode.  rho_j = Kdot_j z + hdot_j, ab2_gar_tangent's right-hand side for tangent j,
//    written (not negated) in resolve's rhs layouts; resolve(rho_j) is then zdot_j.
//
// Layout: one warp per stage knot (instance b, knot t), grid-stride; the warp stages the knot's primal vectors
// x_t, u_t, v_t, lambda_{t+1} once in its slice of shared memory and then loops over the right-hand sides, so z is read
// once per knot and not once per right-hand side.  The terminal record, G0 and g0 get one warp per (instance, rhs).
//  * Gradient: the map "element of the record -> the two vector entries and the kind of product" is built once per
//    CTA from the record layout (lq_record.cuh).  A chunk of right-hand sides' y vectors is staged, then the lanes run
//    over consecutive (rhs, element) pairs, so the stores are coalesced and a short record (C3: 76 doubles) leaves no
//    lane idle.
//  * Rho: tangent records are staged by cp.async in tiles of at most kTile doubles; a record that fits a tile is staged
//    together with the records of the next right-hand sides (as many as fit), and the lanes run over (rhs, row) pairs.
//    Each lane sums its rows in a fixed order (tile by tile, block by block, element by element); the tile boundaries
//    depend on the record length only.
// So right-hand side j's result is bit for bit independent of nrhs and of j's position, and of timing.
// Both kernels have a generalised instantiation (EXT, ab2_gar_rho_many / ab2_gar_grad_many, DESIGN section 2p): the
// vector blocks optional, a per-right-hand-side z staged once per (rhs, knot) beside the shared one, a second term or
// pair without vector blocks, and an addend e, each element still summed in one fixed order.
#include <cuda_runtime.h>

#include "cp_async.cuh"
#include "lq_jacobian.h"
#include "lq_record.cuh"

namespace ab2 {

namespace {
constexpr int kWarps = 8;        // warps per CTA
constexpr int kTile = 512;       // doubles of tangent records one warp stages at a time
constexpr int kVecDoubles = 512; // doubles of z and a chunk of y vectors one warp of the gradient kernel stages
constexpr int kMaxChunk = 16;    // right-hand sides whose y one warp of the gradient kernel stages at once

// ---- gradient records ----
enum : unsigned { G_PAIR = 0, G_HALF = 1, G_SINGLE = 2, G_ZERO = 3 }; // y_a p_b + p_a y_b, half of it, y_a, 0
// a, b: offsets of the two entries in the knot's vector buffer
__device__ __forceinline__ unsigned gentry(int a, int b, unsigned mode) {
  return (unsigned)a | ((unsigned)b << 15) | (mode << 30);
}
// times sgn = +1 or -1 (exact: -1 negates; a pad element stays +0.0).  A pair is rounded as fma(y_a, p_b, p_a y_b), or
// with swap as fma(p_a, y_b, y_a p_b), the order ab2_gar_adjoint's stage gradients have always had.
__device__ __forceinline__ double gvalue(unsigned ent, const double *p, const double *y, double sgn, bool swap) {
  const unsigned mode = ent >> 30;
  const int ia = (int)(ent & 0x7fff), ib = (int)((ent >> 15) & 0x7fff);
  if (mode == G_ZERO)
    return 0.0;
  double s;
  if (mode == G_SINGLE) {
    s = y[ia];
  } else {
    s = swap ? fma(p[ia], y[ib], y[ia] * p[ib]) : fma(y[ia], p[ib], p[ia] * y[ib]);
    if (mode == G_HALF)
      s = 0.5 * s;
  }
  return sgn * s;
}
// The generalised mode's value of one element: Gr^(vec)(y; p) + Gr_K(y2; p2) (two), each pair rounded as the plain
// mode's (sgn = +1, no swap); a vector element of a pair without vectors is 0.
__device__ __forceinline__ double gvalue2(unsigned ent, const double *p, const double *y, bool vec, const double *p2,
                                          const double *y2, bool two) {
  const unsigned mode = ent >> 30;
  double s = mode == G_SINGLE && !vec ? 0.0 : gvalue(ent, p, y, 1.0, false);
  if (two)
    s += mode == G_SINGLE ? 0.0 : gvalue(ent, p2, y2, 1.0, false);
  return s;
}
// Entry k of knot `it`'s vector [x | u | v | l] (k < 2 nx + nu + nc) of the solution-layout vector z, whose row (the
// instance, or j * batch + b) is `row`: x_t sits in row `row` of [.][N+1][nx], the others in [.][N][.].
__device__ __forceinline__ double knot_entry(const double *xs, const double *us, const double *vs, const double *lams,
                                             long it, long row, int k, int nx, int nu, int nc) {
  const int U = nx, V = nx + nu, L = nx + nu + nc;
  return k < U ? xs[(it + row) * nx + k] : k < V ? us[it * nu + k - U] : k < L ? vs[it * nc + k - V]
                                                                             : lams[it * nx + k - L];
}
__device__ __forceinline__ double knot_entry(const SolVec &z, long it, long row, int k, int nx, int nu, int nc) {
  return knot_entry(z.xs, z.us, z.vs, z.lams, it, row, k, nx, nu, nc);
}
// Entry k of row `row`'s terminal vector [x_N | v_N | x_0 | l_0] (k < 2 nx + nct + nc0) of z.
__device__ __forceinline__ double term_entry(const SolVec &z, long row, int k, int nx, int nct, int nc0, int N) {
  if (k < nx)
    return z.xs[(row * (N + 1) + N) * nx + k];
  if (k < nx + nct)
    return z.vsT[row * nct + k - nx];
  if (k < 2 * nx + nct)
    return z.xs[row * (N + 1) * nx + k - nx - nct];
  return z.lam0[row * nc0 + k - 2 * nx - nct];
}

// ---- rho rows from a staged tile holding record elements [e0, e1) ----
// Part of row i of M y (col = false) or of M^T y (col = true) in the tile, for the m x n block M at record offset o.
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
// stage rows [q (nx) | r (nu) | d (nc) | f (nx)]:
//   rho_q = qdot + sym(Qdot) x + Sdot u + Cdot^T v + Adot^T l,  rho_r = rdot + Sdot^T x + sym(Rdot) u + Ddot^T v + Bdot^T l,
//   rho_d = ddot + Cdot x + Ddot u,  rho_f = fdot + Adot x + Bdot u
// vec = false: rho_K, the same rows without the tangent's vector blocks (qdot, rdot, ddot, fdot)
__device__ __forceinline__ double stage_row(const double *tile, int e0, int e1, const StageOffsets &o, int nx, int nu,
                                            int nc, int row, const double *x, const double *u, const double *v,
                                            const double *l, bool vec = true) {
  if (row < nx) {
    const int i = row;
    return (vec ? ve(tile, e0, e1, o.q, i) : 0.0) +
           0.5 * (mv(tile, e0, e1, o.Q, nx, nx, i, false, x) + mv(tile, e0, e1, o.Q, nx, nx, i, true, x)) +
           mv(tile, e0, e1, o.S, nx, nu, i, false, u) + mv(tile, e0, e1, o.C, nc, nx, i, true, v) +
           mv(tile, e0, e1, o.A, nx, nx, i, true, l);
  }
  if (row < nx + nu) {
    const int i = row - nx;
    return (vec ? ve(tile, e0, e1, o.r, i) : 0.0) + mv(tile, e0, e1, o.S, nx, nu, i, true, x) +
           0.5 * (mv(tile, e0, e1, o.R, nu, nu, i, false, u) + mv(tile, e0, e1, o.R, nu, nu, i, true, u)) +
           mv(tile, e0, e1, o.D, nc, nu, i, true, v) + mv(tile, e0, e1, o.B, nx, nu, i, true, l);
  }
  if (row < nx + nu + nc) {
    const int i = row - nx - nu;
    return (vec ? ve(tile, e0, e1, o.d, i) : 0.0) + mv(tile, e0, e1, o.C, nc, nx, i, false, x) +
           mv(tile, e0, e1, o.D, nc, nu, i, false, u);
  }
  const int i = row - nx - nu - nc;
  return (vec ? ve(tile, e0, e1, o.f, i) : 0.0) + mv(tile, e0, e1, o.A, nx, nx, i, false, x) +
         mv(tile, e0, e1, o.B, nx, nu, i, false, u);
}
// terminal rows [q_N (nx) | d_N (nct)]: rho_qN = qdot_N + sym(Qdot_N) x + C_Ndot^T v,  rho_dN = ddot_N + C_Ndot x
__device__ __forceinline__ double term_row(const double *tile, int e0, int e1, const TermOffsets &o, int nx, int nct,
                                           int row, const double *x, const double *v, bool vec = true) {
  if (row < nx)
    return (vec ? ve(tile, e0, e1, o.q, row) : 0.0) +
           0.5 * (mv(tile, e0, e1, o.Q, nx, nx, row, false, x) + mv(tile, e0, e1, o.Q, nx, nx, row, true, x)) +
           mv(tile, e0, e1, o.C, nct, nx, row, true, v);
  const int i = row - nx;
  return (vec ? ve(tile, e0, e1, o.d, i) : 0.0) + mv(tile, e0, e1, o.C, nct, nx, i, false, x);
}

int sm_count() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}
} // namespace

// NEG: a.neg, as a template argument so that the flag costs no register.  EXT: a.ext, the generalised mode (per
// right-hand-side z, a second pair, vector blocks optional); EXT = false is the plain mode's code unchanged.
template <bool NEG, bool EXT>
__global__ void __launch_bounds__(kWarps * 32) jacobian_grad_kernel(const JacobianGradArgs a, int chunk,
                                                                    int warp_doubles) {
  extern __shared__ __align__(16) double smem[];
  const AdjointDims d = a.d;
  const int nx = d.nx, nu = d.nu, nc = d.nc, nct = d.nct, nc0 = d.nc0, N = d.N, B = d.batch, srec = d.srec;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned *map = reinterpret_cast<unsigned *>(smem + (size_t)kWarps * warp_doubles); // [srec] stage, [trec] terminal
  // stage vector buffer [x | u | v | l]; terminal [x_N | v_N | x_0 | l_0]
  const int X = 0, U = nx, V = nx + nu, L = nx + nu + nc, nrow = 2 * nx + nu + nc;
  const int TV = nx, TX0 = nx + nct, TL0 = 2 * nx + nct, tvec = 2 * nx + nct + nc0;
  constexpr double sgn = NEG ? -1.0 : 1.0;
  const StageOffsets so = stage_offsets(nx, nu, nc);
  for (int e = threadIdx.x; e < srec; e += blockDim.x) {
    const RecElem el = stage_elem(so, nx, nu, nc, e);
    const int i = el.row, j = el.col;
    unsigned ent;
    switch (el.blk) {
    case BK_A: ent = gentry(L + i, X + j, G_PAIR); break;  // y_l x^T + l y_x^T
    case BK_B: ent = gentry(L + i, U + j, G_PAIR); break;  // y_l u^T + l y_u^T
    case BK_F: ent = gentry(L + i, 0, G_SINGLE); break;    // y_l
    case BK_Q: ent = gentry(X + i, X + j, G_HALF); break;  // 1/2 (y_x x^T + x y_x^T)
    case BK_S: ent = gentry(X + i, U + j, G_PAIR); break;  // y_x u^T + x y_u^T
    case BK_R: ent = gentry(U + i, U + j, G_HALF); break;  // 1/2 (y_u u^T + u y_u^T)
    case BK_QV: ent = gentry(X + i, 0, G_SINGLE); break;   // y_x
    case BK_RV: ent = gentry(U + i, 0, G_SINGLE); break;   // y_u
    case BK_C: ent = gentry(V + i, X + j, G_PAIR); break;  // y_v x^T + v y_x^T
    case BK_D: ent = gentry(V + i, U + j, G_PAIR); break;  // y_v u^T + v y_u^T
    case BK_DV: ent = gentry(V + i, 0, G_SINGLE); break;   // y_v
    default: ent = gentry(0, 0, G_ZERO);                   // pad
    }
    map[e] = ent;
  }
  const TermOffsets to = term_offsets(nx, nct);
  for (int e = threadIdx.x; e < d.trec; e += blockDim.x) {
    const RecElem el = term_elem(to, nx, nct, e);
    const int i = el.row, j = el.col;
    map[srec + e] = el.blk == BK_Q    ? gentry(X + i, X + j, G_HALF)
                    : el.blk == BK_QV ? gentry(X + i, 0, G_SINGLE)
                    : el.blk == BK_C  ? gentry(TV + i, X + j, G_PAIR)
                                      : gentry(TV + i, 0, G_SINGLE);
  }
  __syncthreads();
  double *pv = smem + (size_t)wid * warp_doubles;
  const long nS = a.stage ? (long)B * N : 0, nT = (a.term || a.G0 || a.g0) ? (long)B * a.nrhs : 0;
  const long w0 = (long)blockIdx.x * kWarps + wid, ws = (long)gridDim.x * kWarps;
  if constexpr (EXT) {
    // stage buffer: [z (nrow) | z2 (nrow) | chunk slots]; the slot of one right-hand side holds y, then z (z_each),
    // y2 and z2 (z2.each).  A shared z or z2 is staged once per knot, a per-right-hand-side one once per (rhs, knot).
    const bool two = a.y2.xs != nullptr, e1 = a.z_each, e2 = two && a.z2.each, vec = a.vec;
    const int slot = nrow * (1 + e1 + (two ? 1 + e2 : 0));
    const SolVec Y{a.yxs, a.yus, a.yvs, a.yvsT, a.ylam0, a.ylams, true};
    const SolVec Z{a.xs, a.us, a.vs, a.vsT, a.lam0, a.lams, e1};
    double *zs = pv, *z2s = pv + nrow, *slots = pv + 2 * nrow;
    for (long it = w0; it < nS + nT; it += ws) {
      if (it < nS) { // stage knot (b, t) = record `it` of every right-hand side
        const long b = it / N;
        for (int k = lane; k < nrow; k += 32) {
          if (!e1)
            zs[k] = knot_entry(Z, it, b, k, nx, nu, nc);
          if (two && !e2)
            z2s[k] = knot_entry(a.z2, it, b, k, nx, nu, nc);
        }
        for (int j0 = 0; j0 < a.nrhs; j0 += chunk) {
          const int R = a.nrhs - j0 < chunk ? a.nrhs - j0 : chunk;
          for (int p = lane; p < R * nrow; p += 32) {
            const int g = p / nrow, k = p - g * nrow;
            const long jit = (long)(j0 + g) * nS + it, jb = jit / N; // record and row (j * batch + b) of rhs j0 + g
            double *sl = slots + g * slot + k;
            sl[0] = knot_entry(Y, jit, jb, k, nx, nu, nc);
            if (e1)
              sl[nrow] = knot_entry(Z, jit, jb, k, nx, nu, nc);
            if (two)
              sl[(1 + e1) * nrow] = knot_entry(a.y2, jit, jb, k, nx, nu, nc);
            if (e2)
              sl[(2 + e1) * nrow] = knot_entry(a.z2, jit, jb, k, nx, nu, nc);
          }
          __syncwarp();
          double *out = a.stage + ((long)j0 * nS + it) * srec;
          const long rstride = nS * srec;
          int g = 0, e = lane;
          while (e >= srec) {
            e -= srec;
            ++g;
          }
          for (int p = lane; p < R * srec; p += 32) {
            const double *sl = slots + g * slot, *y2 = sl + (1 + e1) * nrow;
            out[g * rstride + e] = gvalue2(map[e], e1 ? sl + nrow : zs, sl, vec, e2 ? y2 + nrow : z2s, y2, two);
            e += 32;
            while (e >= srec) {
              e -= srec;
              ++g;
            }
          }
          __syncwarp(); // the slots are overwritten next
        }
      } else { // (instance b, rhs j): terminal record, G0, g0; buffers [z | y | z2 | y2], each [x_N | v_N | x_0 | l_0]
        const long jb = it - nS, b = jb % B, r1 = e1 ? jb : b, r2 = e2 ? jb : b;
        double *yv = pv + tvec, *p2 = pv + 2 * tvec, *y2 = pv + 3 * tvec;
        for (int k = lane; k < tvec; k += 32) {
          pv[k] = term_entry(Z, r1, k, nx, nct, nc0, N);
          yv[k] = term_entry(Y, jb, k, nx, nct, nc0, N);
          if (two) {
            p2[k] = term_entry(a.z2, r2, k, nx, nct, nc0, N);
            y2[k] = term_entry(a.y2, jb, k, nx, nct, nc0, N);
          }
        }
        __syncwarp();
        if (a.term)
          for (int e = lane; e < d.trec; e += 32)
            a.term[jb * d.trec + e] = gvalue2(map[srec + e], pv, yv, vec, p2, y2, two);
        if (a.G0)
          for (int e = lane; e < nc0 * nx; e += 32) {
            const int r = e % nc0, c = e / nc0;
            double v = fma(yv[TL0 + r], pv[TX0 + c], pv[TL0 + r] * yv[TX0 + c]);
            if (two)
              v += fma(y2[TL0 + r], p2[TX0 + c], p2[TL0 + r] * y2[TX0 + c]);
            a.G0[jb * nc0 * nx + e] = v;
          }
        if (a.g0)
          for (int i = lane; i < nc0; i += 32)
            a.g0[jb * nc0 + i] = vec ? yv[TL0 + i] : 0.0;
        __syncwarp();
      }
    }
  } else {
    for (long it = w0; it < nS + nT; it += ws) {
      if (it < nS) { // stage knot (b, t) = record `it` of every right-hand side
        const long b = it / N;
        double *yv = pv + nrow;
        for (int k = lane; k < nrow; k += 32)
          pv[k] = k < U ? a.xs[(it + b) * nx + k] : k < V ? a.us[it * nu + k - U] : k < L ? a.vs[it * nc + k - V]
                                                                                         : a.lams[it * nx + k - L];
        for (int j0 = 0; j0 < a.nrhs; j0 += chunk) {
          const int R = a.nrhs - j0 < chunk ? a.nrhs - j0 : chunk;
          for (int p = lane; p < R * nrow; p += 32) {
            const int g = p / nrow, k = p - g * nrow;
            const long jit = (long)(j0 + g) * nS + it, jb = jit / N; // record and row (j * batch + b) of rhs j0 + g
            yv[p] = k < U ? a.yxs[(jit + jb) * nx + k] : k < V ? a.yus[jit * nu + k - U]
                                                   : k < L ? a.yvs[jit * nc + k - V] : a.ylams[jit * nx + k - L];
          }
          __syncwarp();
          double *out = a.stage + ((long)j0 * nS + it) * srec;
          const long rstride = nS * srec;
          int g = 0, e = lane;
          while (e >= srec) {
            e -= srec;
            ++g;
          }
          for (int p = lane; p < R * srec; p += 32) {
            out[g * rstride + e] = gvalue(map[e], pv, yv + g * nrow, sgn, NEG);
            e += 32;
            while (e >= srec) {
              e -= srec;
              ++g;
            }
          }
          __syncwarp(); // yv is overwritten next
        }
      } else { // (instance b, rhs j): terminal record, G0, g0
        const long jb = it - nS, b = jb % B;
        double *yv = pv + tvec;
        for (int k = lane; k < tvec; k += 32) {
          double p, y;
          if (k < TV) {
            p = a.xs[(b * (N + 1) + N) * nx + k];
            y = a.yxs[(jb * (N + 1) + N) * nx + k];
          } else if (k < TX0) {
            p = a.vsT[b * nct + k - TV];
            y = a.yvsT[jb * nct + k - TV];
          } else if (k < TL0) {
            p = a.xs[b * (N + 1) * nx + k - TX0];
            y = a.yxs[jb * (N + 1) * nx + k - TX0];
          } else {
            p = a.lam0[b * nc0 + k - TL0];
            y = a.ylam0[jb * nc0 + k - TL0];
          }
          pv[k] = p;
          yv[k] = y;
        }
        __syncwarp();
        if (a.term)
          for (int e = lane; e < d.trec; e += 32)
            a.term[jb * d.trec + e] = gvalue(map[srec + e], pv, yv, sgn, false);
        if (a.G0) // dG0 = y_l0 x_0^T + l_0 y_x0^T, column-major [nc0][nx]
          for (int e = lane; e < nc0 * nx; e += 32) {
            const int r = e % nc0, c = e / nc0;
            const double v = fma(yv[TL0 + r], pv[TX0 + c], pv[TL0 + r] * yv[TX0 + c]);
            a.G0[jb * nc0 * nx + e] = sgn * v;
          }
        if (a.g0)
          for (int i = lane; i < nc0; i += 32)
            a.g0[jb * nc0 + i] = sgn * yv[TL0 + i];
        __syncwarp();
      }
    }
  }
}

// ONE: nrhs = 1 (ab2_gar_tangent), where the right-hand-side loop is a single pass and 4 CTAs per SM fit the registers.
// EXT: a.ext, the generalised mode (per right-hand-side z, a second term, vector blocks optional, e); EXT = false is the
// plain mode's code unchanged.
template <bool ONE, bool EXT>
__global__ void __launch_bounds__(kWarps * 32, ONE ? 4 : 3) jacobian_rhs_kernel(const JacobianRhsArgs a, int slice, int group,
                                                                      int warp_doubles) {
  extern __shared__ __align__(16) double smem[];
  const AdjointDims d = a.d;
  const int nx = d.nx, nu = d.nu, nc = d.nc, nct = d.nct, nc0 = d.nc0, N = d.N, B = d.batch;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  double *tile = smem + (size_t)wid * warp_doubles;
  double *vec = tile + kTile;
  const StageOffsets so = stage_offsets(nx, nu, nc);
  const TermOffsets to = term_offsets(nx, nct);
  const int nrow = 2 * nx + nu + nc;
  const long nS = (long)B * N, items = nS + (long)B * a.nrhs;
  const long w0 = (long)blockIdx.x * kWarps + wid, ws = (long)gridDim.x * kWarps;
  if constexpr (EXT) {
    // stage buffer: [z (nrow) | z2 (nrow) | the group's per-rhs z or z2 (group * nrow) | acc (group * nrow)].  A shared
    // z or z2 is staged once per knot, a per-right-hand-side one once per (rhs, knot).  Each row sums the first term
    // tile by tile, then the second term tile by tile, then the G0 products, then e: a fixed order.
    const bool two = a.two, e1 = a.z_each, e2 = two && a.z2.each, vec1 = a.vec;
    const SolVec Z{a.xs, a.us, a.vs, a.vsT, a.lam0, a.lams, e1};
    const SolVec &Z2 = a.z2, &E = a.e;
    const int nv = nx + nu + nc; // the offset of l in a knot vector
    for (long it = w0; it < items; it += ws) {
      if (it < nS) { // stage knot (b, t) = record `it` of every right-hand side
        const long b = it / N;
        const int t = (int)(it - b * N);
        double *zs = vec, *z2s = zs + nrow, *pd = z2s + nrow, *acc = pd + group * nrow;
        for (int k = lane; k < nrow; k += 32) {
          if (!e1)
            zs[k] = knot_entry(Z, it, b, k, nx, nu, nc);
          if (two && !e2)
            z2s[k] = knot_entry(Z2, it, b, k, nx, nu, nc);
        }
        __syncwarp();
        for (int j0 = 0; j0 < a.nrhs; j0 += group) {
          const int R = a.nrhs - j0 < group ? a.nrhs - j0 : group;
          for (int p = lane; p < R * nrow; p += 32) {
            acc[p] = 0.0;
            if (e1) {
              const int g = p / nrow;
              const long jit = (long)(j0 + g) * nS + it;
              pd[p] = knot_entry(Z, jit, jit / N, p - g * nrow, nx, nu, nc);
            }
          }
          // term 1, then term 2: the tangent records of the group, tile by tile (the wait's __syncwarp also publishes pd)
          for (int term = 0; term < (two ? 2 : 1); ++term) {
            const double *rec = term ? a.stage2 : a.stage;
            const bool each = term ? e2 : e1;
            if (!rec)
              continue;
            if (term && e2) {
              __syncwarp(); // term 1 has read pd
              for (int p = lane; p < R * nrow; p += 32) {
                const int g = p / nrow;
                const long jit = (long)(j0 + g) * nS + it;
                pd[p] = knot_entry(Z2, jit, jit / N, p - g * nrow, nx, nu, nc);
              }
            }
            for (int e0 = 0; e0 < d.srec; e0 += slice) {
              const int eh = e0 + slice < d.srec ? e0 + slice : d.srec;
              for (int g = 0; g < R; ++g)
                stage_copy(tile + g * slice, rec + ((long)(j0 + g) * nS + it) * d.srec + e0, eh - e0, lane);
              cp_wait_all();
              __syncwarp();
              for (int p = lane; p < R * nrow; p += 32) {
                const int g = p / nrow;
                const double *z = each ? pd + g * nrow : term ? z2s : zs;
                acc[p] += stage_row(tile + g * slice, e0, eh, so, nx, nu, nc, p - g * nrow, z, z + nx, z + nx + nu,
                                    z + nv, term ? false : vec1);
              }
              __syncwarp(); // the tile is overwritten next
            }
          }
          for (int p = lane; p < R * nrow; p += 32) {
            const int g = p / nrow, r = p - g * nrow;
            const long jit = (long)(j0 + g) * nS + it, jb = jit / N; // record and row (j * batch + b) of rhs j0 + g
            double s = acc[p];
            if (r < nx) {
              if (t == 0) { // + G0dot^T lambda_0 of each term, G0dot column-major [nc0][nx]
                for (int term = 0; term < (two ? 2 : 1); ++term) {
                  const double *G = term ? a.G02 : a.G0;
                  const SolVec &z = term ? Z2 : Z;
                  if (!G)
                    continue;
                  const double *Gc = G + jb * nc0 * nx + (long)r * nc0, *l0 = z.lam0 + ((term ? e2 : e1) ? jb : b) * nc0;
                  double gs = 0.0;
                  for (int k = 0; k < nc0; ++k)
                    gs = fma(Gc[k], l0[k], gs);
                  s += gs;
                }
              }
              const long o = (jit + jb) * nx + r;
              a.q[o] = E.xs ? s + E.xs[o] : s;
            } else if (r < nx + nu) {
              const long o = jit * nu + r - nx;
              a.r[o] = E.xs ? s + E.us[o] : s;
            } else if (r < nv) {
              const long o = jit * nc + r - nx - nu;
              a.dv[o] = E.xs ? s + E.vs[o] : s;
            } else {
              const long o = jit * nx + r - nv;
              a.f[o] = E.xs ? s + E.lams[o] : s;
            }
          }
          __syncwarp(); // acc and pd are overwritten next
        }
      } else { // (instance b, rhs j): rows [q_N (nx) | d_N (nct) | g0 (nc0)]
        const long jb = it - nS, b = jb % B, r1 = e1 ? jb : b, r2 = e2 ? jb : b;
        const int trows = nx + nct + nc0;
        double *x = vec, *v = x + nx, *x2 = v + nct, *v2 = x2 + nx, *acc = v2 + nct;
        for (int k = lane; k < nx + nct; k += 32) {
          vec[k] = k < nx ? Z.xs[(r1 * (N + 1) + N) * nx + k] : Z.vsT[r1 * nct + k - nx];
          if (two)
            x2[k] = k < nx ? Z2.xs[(r2 * (N + 1) + N) * nx + k] : Z2.vsT[r2 * nct + k - nx];
        }
        for (int r = lane; r < trows; r += 32)
          acc[r] = 0.0;
        __syncwarp();
        for (int term = 0; term < (two ? 2 : 1); ++term) {
          const double *rec = term ? a.term2 : a.term;
          if (!rec)
            continue;
          for (int e0 = 0; e0 < d.trec; e0 += kTile) {
            const int eh = e0 + kTile < d.trec ? e0 + kTile : d.trec;
            stage_copy(tile, rec + jb * d.trec + e0, eh - e0, lane);
            cp_wait_all();
            __syncwarp();
            for (int r = lane; r < nx + nct; r += 32)
              acc[r] += term ? term_row(tile, e0, eh, to, nx, nct, r, x2, v2, false)
                             : term_row(tile, e0, eh, to, nx, nct, r, x, v, vec1);
            __syncwarp();
          }
        }
        for (int r = lane; r < trows; r += 32) {
          double s = acc[r];
          if (r < nx) {
            if (N == 0) // x_0 = x_N: + G0dot^T lambda_0 of each term
              for (int term = 0; term < (two ? 2 : 1); ++term) {
                const double *G = term ? a.G02 : a.G0;
                if (!G)
                  continue;
                const double *Gc = G + jb * nc0 * nx, *l0 = (term ? Z2 : Z).lam0 + (term ? r2 : r1) * nc0;
                double gs = 0.0;
                for (int k = 0; k < nc0; ++k)
                  gs = fma(Gc[(long)r * nc0 + k], l0[k], gs);
                s += gs;
              }
            const long o = (jb * (N + 1) + N) * nx + r;
            a.q[o] = E.xs ? s + E.xs[o] : s;
          } else if (r < nx + nct) {
            const long o = jb * nct + r - nx;
            a.dN[o] = E.xs ? s + E.vsT[o] : s;
          } else { // rho_g0 = g0dot (with vectors) + G0dot x_0 of each term
            const int i = r - nx - nct;
            if (vec1 && a.g0)
              s += a.g0[jb * nc0 + i];
            for (int term = 0; term < (two ? 2 : 1); ++term) {
              const double *G = term ? a.G02 : a.G0;
              if (!G)
                continue;
              const double *Gc = G + jb * nc0 * nx, *x0 = (term ? Z2 : Z).xs + (term ? r2 : r1) * (N + 1) * nx;
              double gs = 0.0;
              for (int c = 0; c < nx; ++c)
                gs = fma(Gc[i + (long)c * nc0], x0[c], gs);
              s += gs;
            }
            const long o = jb * nc0 + i;
            a.g0out[o] = E.xs ? s + E.lam0[o] : s;
          }
        }
        __syncwarp();
      }
    }
  } else {
    for (long it = w0; it < items; it += ws) {
      if (it < nS) { // stage knot (b, t) = record `it` of every right-hand side
        const long b = it / N;
        const int t = (int)(it - b * N);
        double *x = vec, *u = x + nx, *v = u + nu, *l = v + nc, *acc = l + nx;
        for (int k = lane; k < nrow; k += 32)
          vec[k] = k < nx ? a.xs[(it + b) * nx + k] : k < nx + nu ? a.us[it * nu + k - nx]
                   : k < nx + nu + nc ? a.vs[it * nc + k - nx - nu] : a.lams[it * nx + k - nx - nu - nc];
        __syncwarp();
        for (int j0 = 0; j0 < (ONE ? 1 : a.nrhs); j0 += group) {
          const int R = ONE ? 1 : (a.nrhs - j0 < group ? a.nrhs - j0 : group);
          for (int p = lane; p < R * nrow; p += 32)
            acc[p] = 0.0;
          if (a.stage) {
            for (int e0 = 0; e0 < d.srec; e0 += slice) {
              const int e1 = e0 + slice < d.srec ? e0 + slice : d.srec;
              for (int g = 0; g < R; ++g)
                stage_copy(tile + g * slice, a.stage + ((long)(j0 + g) * nS + it) * d.srec + e0, e1 - e0, lane);
              cp_wait_all();
              __syncwarp();
              for (int p = lane; p < R * nrow; p += 32) {
                const int g = p / nrow;
                acc[p] += stage_row(tile + g * slice, e0, e1, so, nx, nu, nc, p - g * nrow, x, u, v, l);
              }
              __syncwarp(); // the tile is overwritten next
            }
          }
          for (int p = lane; p < R * nrow; p += 32) {
            const int g = p / nrow, r = p - g * nrow;
            const long jit = (long)(j0 + g) * nS + it, jb = jit / N; // record and row (j * batch + b) of rhs j0 + g
            double s = acc[p];
            if (r < nx) {
              if (t == 0 && a.G0) { // + G0dot^T lambda_0, G0dot column-major [nc0][nx]
                const double *G = a.G0 + jb * nc0 * nx + (long)r * nc0, *l0 = a.lam0 + b * nc0;
                double gs = 0.0;
                for (int k = 0; k < nc0; ++k)
                  gs = fma(G[k], l0[k], gs);
                s += gs;
              }
              a.q[(jit + jb) * nx + r] = s;
            } else if (r < nx + nu) {
              a.r[jit * nu + r - nx] = s;
            } else if (r < nx + nu + nc) {
              a.dv[jit * nc + r - nx - nu] = s;
            } else {
              a.f[jit * nx + r - nx - nu - nc] = s;
            }
          }
        }
        __syncwarp(); // the vectors are overwritten next
      } else { // (instance b, rhs j): rows [q_N (nx) | d_N (nct) | g0 (nc0)]
        const long jb = it - nS, b = jb % B;
        const int trows = nx + nct + nc0;
        double *x = vec, *v = x + nx, *acc = v + nct;
        for (int k = lane; k < nx + nct; k += 32)
          vec[k] = k < nx ? a.xs[(b * (N + 1) + N) * nx + k] : a.vsT[b * nct + k - nx];
        for (int r = lane; r < trows; r += 32)
          acc[r] = 0.0;
        __syncwarp();
        if (a.term) {
          for (int e0 = 0; e0 < d.trec; e0 += kTile) {
            const int e1 = e0 + kTile < d.trec ? e0 + kTile : d.trec;
            stage_copy(tile, a.term + jb * d.trec + e0, e1 - e0, lane);
            cp_wait_all();
            __syncwarp();
            for (int r = lane; r < nx + nct; r += 32)
              acc[r] += term_row(tile, e0, e1, to, nx, nct, r, x, v);
            __syncwarp();
          }
        }
        const double *G = a.G0 ? a.G0 + jb * nc0 * nx : nullptr, *l0 = a.lam0 + b * nc0, *x0 = a.xs + b * (N + 1) * nx;
        for (int r = lane; r < trows; r += 32) {
          double s = acc[r];
          if (r < nx) {
            if (N == 0 && G) { // x_0 = x_N: + G0dot^T lambda_0
              double gs = 0.0;
              for (int k = 0; k < nc0; ++k)
                gs = fma(G[(long)r * nc0 + k], l0[k], gs);
              s += gs;
            }
            a.q[(jb * (N + 1) + N) * nx + r] = s;
          } else if (r < nx + nct) {
            a.dN[jb * nct + r - nx] = s;
          } else { // rho_g0 = g0dot + G0dot x_0
            const int i = r - nx - nct;
            if (a.g0)
              s += a.g0[jb * nc0 + i];
            if (G) {
              double gs = 0.0;
              for (int c = 0; c < nx; ++c)
                gs = fma(G[i + (long)c * nc0], x0[c], gs);
              s += gs;
            }
            a.g0out[jb * nc0 + i] = s;
          }
        }
        __syncwarp();
      }
    }
  }
}

cudaError_t launch_jacobian_grad(const JacobianGradArgs &a, cudaStream_t st) {
  const AdjointDims &d = a.d;
  const long items = (a.stage ? (long)d.batch * d.N : 0) + ((a.term || a.G0 || a.g0) ? (long)d.batch * a.nrhs : 0);
  if (a.nrhs <= 0 || items <= 0)
    return cudaSuccess;
  const int nrow = 2 * d.nx + d.nu + d.nc, tvec = 2 * d.nx + d.nct + d.nc0;
  // plain: [z | chunk y]; generalised: [z | z2 | chunk slots of y, z (z_each), y2, z2 (z2.each)], terminal [z|y|z2|y2]
  const bool two = a.ext && a.y2.xs;
  const int shared = a.ext ? 2 * nrow : nrow, slot = nrow * (1 + (a.ext && a.z_each) + (two ? 1 + a.z2.each : 0));
  int chunk = (kVecDoubles - shared) / slot;
  chunk = chunk < 1 ? 1 : (chunk > kMaxChunk ? kMaxChunk : chunk);
  chunk = chunk < a.nrhs ? chunk : a.nrhs;
  const int tneed = (a.ext ? 4 : 2) * tvec;
  int warp_doubles = shared + slot * chunk > tneed ? shared + slot * chunk : tneed;
  warp_doubles = (warp_doubles + 1) & ~1;
  const size_t smem = (size_t)warp_doubles * kWarps * sizeof(double) + (size_t)(d.srec + d.trec) * sizeof(unsigned);
  void (*kernel)(const JacobianGradArgs, int, int) = a.ext ? jacobian_grad_kernel<false, true>
                                                     : a.neg ? jacobian_grad_kernel<true, false>
                                                             : jacobian_grad_kernel<false, false>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess)
    return e;
  int per_sm = 1;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kWarps * 32, smem);
  if (e != cudaSuccess)
    return e;
  long grid = (items + kWarps - 1) / kWarps;
  const long full = (long)sm_count() * (per_sm > 0 ? per_sm : 1);
  grid = grid < full ? grid : full;
  kernel<<<(int)grid, kWarps * 32, smem, st>>>(a, chunk, warp_doubles);
  return cudaGetLastError();
}

cudaError_t launch_jacobian_rhs(const JacobianRhsArgs &a, cudaStream_t st) {
  const AdjointDims &d = a.d;
  const long items = (long)d.batch * d.N + (long)d.batch * a.nrhs;
  if (a.nrhs <= 0 || items <= 0)
    return cudaSuccess;
  // a stage record that fits the tile is staged whole, together with those of the next right-hand sides
  int slice = d.srec < kTile ? d.srec : kTile;
  slice = (slice + 1) & ~1; // keeps every record's slot 16-byte aligned
  if (slice < 2)
    slice = 2;
  int group = d.srec <= kTile ? kTile / slice : 1;
  group = group < a.nrhs ? group : a.nrhs;
  const int nrow = 2 * d.nx + d.nu + d.nc, trows = d.nx + d.nct + d.nc0;
  // plain: [z | acc], terminal [x_N | v_N | acc]; generalised: [z | z2 | pd | acc], terminal [x_N | v_N | x2_N | v2_N | acc]
  const int svecs = a.ext ? 2 * nrow + 2 * group * nrow : nrow + group * nrow;
  const int tvecs = (a.ext ? 2 : 1) * (d.nx + d.nct) + trows;
  const int vecs = svecs > tvecs ? svecs : tvecs;
  const int warp_doubles = (kTile + vecs + 1) & ~1;
  const size_t smem = (size_t)warp_doubles * kWarps * sizeof(double);
  void (*kernel)(const JacobianRhsArgs, int, int, int) = a.ext ? jacobian_rhs_kernel<false, true>
                                                         : a.nrhs == 1 ? jacobian_rhs_kernel<true, false>
                                                                       : jacobian_rhs_kernel<false, false>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess)
    return e;
  int per_sm = 1;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kWarps * 32, smem);
  if (e != cudaSuccess)
    return e;
  long grid = (items + kWarps - 1) / kWarps;
  const long full = (long)sm_count() * (per_sm > 0 ? per_sm : 1);
  grid = grid < full ? grid : full;
  kernel<<<(int)grid, kWarps * 32, smem, st>>>(a, slice, group, warp_doubles);
  return cudaGetLastError();
}

} // namespace ab2
