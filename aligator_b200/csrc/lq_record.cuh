// lq_record.cuh -- the knot-record layouts of gar.h, defined once for every program that reads or writes a record:
// where each block of a stage record [A | B | f | Q | S | R | q | r | C | D | d | pad] and of a terminal record
// [Q | q | C | d] starts, the parametric tails behind them, the record lengths, the
// triangle-packed stage record of ab2_gar_sweep_host_sym, which block, row and column an element of a record is, and
// which ring slot holds a knot's record.  Matrices are column-major.  Everything is
// constexpr, so compile-time shapes fold it.  Includable from plain C++ (the emulation library).
#pragma once

#if defined(__CUDACC__)
#define AB2_REC_HD __host__ __device__ __forceinline__
#else
#define AB2_REC_HD inline
#endif

namespace ab2 {

struct StageOffsets {
  int A, B, f, Q, S, R, q, r, C, D, d, end; // block starts; end = unpadded length
};
struct TermOffsets {
  int Q, q, C, d, end;
};
// the parametric tail (nth > 0) behind a record's `end`: [Gx | Gu | Gv | Gth | gamma] of a stage record,
// [Gx | Gv | Gth | gamma] of a terminal one (Gu = Gv there)
struct TailOffsets {
  int Gx, Gu, Gv, Gth, gamma, end;
};

AB2_REC_HD constexpr StageOffsets stage_offsets(int nx, int nu, int nc) {
  StageOffsets o{};
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
AB2_REC_HD constexpr TermOffsets term_offsets(int nx, int nct) {
  TermOffsets o{};
  o.Q = 0;
  o.q = nx * nx;
  o.C = o.q + nx;
  o.d = o.C + nct * nx;
  o.end = o.d + nct;
  return o;
}
AB2_REC_HD constexpr TailOffsets stage_tail(const StageOffsets &o, int nx, int nu, int nc, int nth) {
  TailOffsets t{};
  t.Gx = o.end;
  t.Gu = t.Gx + nx * nth;
  t.Gv = t.Gu + nu * nth;
  t.Gth = t.Gv + nc * nth;
  t.gamma = t.Gth + nth * nth;
  t.end = t.gamma + nth;
  return t;
}
AB2_REC_HD constexpr TailOffsets term_tail(const TermOffsets &o, int nx, int nct, int nth) {
  TailOffsets t{};
  t.Gx = o.end;
  t.Gu = t.Gv = t.Gx + nx * nth;
  t.Gth = t.Gv + nct * nth;
  t.gamma = t.Gth + nth * nth;
  t.end = t.gamma + nth;
  return t;
}

// stored length of a stage record: padded to even, so every record starts 16-byte aligned for the bulk copies
AB2_REC_HD constexpr int stage_pad(int end) { return (end + 1) & ~1; }
AB2_REC_HD constexpr int stage_record_len(int nx, int nu, int nc, int nth = 0) {
  return stage_pad(stage_tail(stage_offsets(nx, nu, nc), nx, nu, nc, nth).end);
}
AB2_REC_HD constexpr int term_record_len(int nx, int nct, int nth = 0) {
  return term_tail(term_offsets(nx, nct), nx, nct, nth).end;
}

// storage slot of knot t's stage record in a ring of N records whose first knot is at slot `head` (cycle_append)
AB2_REC_HD int ring_slot(int t, int head, int N) { return t + head >= N ? t + head - N : t + head; }

// ---- the triangle-packed stage record (ab2_gar_sweep_host_sym): [A | B | f | tri(Q) | S | tri(R) | q | r | C | D | d],
// no padding; tri(X) = the lower triangle column by column (column j holds rows j..n-1)
AB2_REC_HD constexpr int stage_sym_len(int nx, int nu, int nc) {
  return stage_offsets(nx, nu, nc).end - nx * (nx - 1) / 2 - nu * (nu - 1) / 2;
}
// slot, in the triangle-packed record, of element e of the full record; both elements of a symmetric pair of Q or R
// map to the slot of the lower one
AB2_REC_HD int sym_source(int e, int nx, int nu, int nc) {
  const int off_q = stage_offsets(nx, nu, nc).Q, tq = nx * (nx + 1) / 2, tr = nu * (nu + 1) / 2;
  if (e < off_q)
    return e;
  e -= off_q;
  if (e < nx * nx) {
    int i = e % nx, j = e / nx;
    if (i < j) {
      const int t = i;
      i = j;
      j = t;
    }
    return off_q + j * nx - j * (j - 1) / 2 + (i - j);
  }
  e -= nx * nx;
  if (e < nx * nu)
    return off_q + tq + e;
  e -= nx * nu;
  if (e < nu * nu) {
    int i = e % nu, j = e / nu;
    if (i < j) {
      const int t = i;
      i = j;
      j = t;
    }
    return off_q + tq + nx * nu + j * nu - j * (j - 1) / 2 + (i - j);
  }
  e -= nu * nu;
  return off_q + tq + nx * nu + tr + e; // q, r, C, D, d
}

// the blocks of a stage record, in storage order; the terminal record uses BK_Q, BK_QV, BK_C, BK_DV
enum : int { BK_A, BK_B, BK_F, BK_Q, BK_S, BK_R, BK_QV, BK_RV, BK_C, BK_D, BK_DV, BK_PAD };
struct RecElem {
  int blk, row, col; // a vector block has col = 0
};

AB2_REC_HD RecElem mat_elem(int blk, int r, int m) { return RecElem{blk, r % m, r / m}; }

// element e of a stage record
AB2_REC_HD RecElem stage_elem(const StageOffsets &o, int nx, int nu, int nc, int e) {
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
AB2_REC_HD RecElem term_elem(const TermOffsets &o, int nx, int nct, int e) {
  if (e < o.q)
    return mat_elem(BK_Q, e - o.Q, nx);
  if (e < o.C)
    return RecElem{BK_QV, e - o.q, 0};
  if (e < o.d)
    return mat_elem(BK_C, e - o.C, nct);
  return RecElem{BK_DV, e - o.d, 0};
}

} // namespace ab2
