// lq_record.cuh -- the knot-record layouts of gar.h, for the Jacobian kernels (lq_jacobian.cu): where each block of a
// stage record [A | B | f | Q | S | R | q | r | C | D | d | pad] and of a terminal record [Q | q | C | d] starts, and
// which block, row and column an element of a record is.  Matrices are column-major.
#pragma once

#include <cuda_runtime.h>

namespace ab2 {

struct StageOffsets {
  int A, B, f, Q, S, R, q, r, C, D, d, end; // block starts; end = unpadded length
};
struct TermOffsets {
  int Q, q, C, d, end;
};

__host__ __device__ __forceinline__ StageOffsets stage_offsets(int nx, int nu, int nc) {
  StageOffsets o;
  o.A = 0;
  o.B = o.A + nx * nx;
  o.f = o.B + nx * nu;
  o.Q = o.f + nx;
  o.S = o.Q + nx * nx;
  o.R = o.S + nx * nu;
  o.q = o.R + nu * nu;
  o.r = o.q + nx;
  o.C = o.r + nu;
  o.D = o.C + nc * nx;
  o.d = o.D + nc * nu;
  o.end = o.d + nc;
  return o;
}
__host__ __device__ __forceinline__ TermOffsets term_offsets(int nx, int nct) {
  TermOffsets o;
  o.Q = 0;
  o.q = nx * nx;
  o.C = o.q + nx;
  o.d = o.C + nct * nx;
  o.end = o.d + nct;
  return o;
}

// the blocks of a stage record, in storage order; the terminal record uses BK_Q, BK_QV, BK_C, BK_DV
enum : int { BK_A, BK_B, BK_F, BK_Q, BK_S, BK_R, BK_QV, BK_RV, BK_C, BK_D, BK_DV, BK_PAD };
struct RecElem {
  int blk, row, col; // a vector block has col = 0
};

__host__ __device__ __forceinline__ RecElem mat_elem(int blk, int r, int m) { return RecElem{blk, r % m, r / m}; }

// element e of a stage record
__host__ __device__ __forceinline__ RecElem stage_elem(const StageOffsets &o, int nx, int nu, int nc, int e) {
  if (e < o.B)
    return mat_elem(BK_A, e - o.A, nx);
  if (e < o.f)
    return mat_elem(BK_B, e - o.B, nx);
  if (e < o.Q)
    return RecElem{BK_F, e - o.f, 0};
  if (e < o.S)
    return mat_elem(BK_Q, e - o.Q, nx);
  if (e < o.R)
    return mat_elem(BK_S, e - o.S, nx);
  if (e < o.q)
    return mat_elem(BK_R, e - o.R, nu);
  if (e < o.r)
    return RecElem{BK_QV, e - o.q, 0};
  if (e < o.C)
    return RecElem{BK_RV, e - o.r, 0};
  if (e < o.D)
    return mat_elem(BK_C, e - o.C, nc);
  if (e < o.d)
    return mat_elem(BK_D, e - o.D, nc);
  if (e < o.end)
    return RecElem{BK_DV, e - o.d, 0};
  return RecElem{BK_PAD, 0, 0};
}
// element e of a terminal record (C and d have nct rows)
__host__ __device__ __forceinline__ RecElem term_elem(const TermOffsets &o, int nx, int nct, int e) {
  if (e < o.q)
    return mat_elem(BK_Q, e - o.Q, nx);
  if (e < o.C)
    return RecElem{BK_QV, e - o.q, 0};
  if (e < o.d)
    return mat_elem(BK_C, e - o.C, nct);
  return RecElem{BK_DV, e - o.d, 0};
}

} // namespace ab2
