// riccati_group.cuh -- the batched Riccati sweep as a *group program*.
//
// One group of G lanes (G = 8, 16 or 32: a warp or a sub-warp) owns one problem
// instance and walks its horizon: terminal knot -> stage knots N-1..0 (backward
// factorisation) -> initial saddle system -> knots 0..N (forward rollout).
//
// What it computes is aligator's gar::ProximalRiccatiSolver::backward/forward
// (gar/proximal-riccati.hxx:34-76, gar/riccati-kernel.hxx:105-377) with the
// Bunch-Kaufman factorisation of core/bunchkaufman.hpp:22-169, 451-518; HOW is
// GPU-first and shares nothing with the reference's Eigen code:
//
//  * lane-per-column mapping: lane j owns column j of  M = [A | B | f]
//    (nx x (nx+nu+1)); one knot step is
//        W  = V' M                         (V' broadcast from shared memory)
//        H  = [[Q S q],[S^T R r]] + [A B]^T W     ([A B] broadcast)
//        KKT = [[Rhat, D^T],[D, -mu I]] -> Bunch-Kaufman, cooperative, in smem
//        [K k; Z z] = -KKT^-1 [Shat^T rhat; C d]  (each lane solves its column)
//        [Ahat a] = [A f] + B [K k],   [Vxx vx] = [Qhat qhat] + [Shat C^T][K k; Z z]
//    so every lane keeps its columns in registers and the only shared-memory
//    traffic is warp-wide broadcast reads;
//  * the knot record (one contiguous [A|B|f|Q|S|R|q|r|C|D|d] block in HBM) is
//    staged by two TMA bulk copies (cp.async.bulk + mbarrier) issued one knot
//    ahead; V' never leaves the chip between knots;
//  * fp64 throughout (the reference's Scalar, context.hpp:9).
//
// The same source compiles for the host (g++), where a "group" is G std::threads
// and sync() is a std::barrier: tests/test_group_emulation.py runs the exact
// index arithmetic below on the CPU before any GPU time is spent.
#pragma once

#include <cmath>
#include <cstddef>
#include <cstdint>
#include <utility>

#include "lq_record.cuh"
#include "vxx_layout.h"

#if defined(__CUDACC__)
#define AB2_HD __host__ __device__ __forceinline__
#define AB2_D __device__ __forceinline__ // group-program code: device only under nvcc
#define AB2_UNROLL _Pragma("unroll")
#else
#define AB2_HD inline
#define AB2_D inline
#define AB2_UNROLL
#endif

namespace ab2 {

// status bits (per instance)
enum : int { ST_OK = 0, ST_STAGE_FACTOR_FAILED = 1, ST_INIT_FACTOR_FAILED = 2 };

struct SweepParams {
  int N;     // horizon: N stage knots + 1 terminal knot
  int nct;   // terminal-knot constraint rows
  int nc0;   // initial-condition rows
  int batch; // instances
  double mueq;
  int do_bwd, do_fwd;
  // inputs
  const double *stage; // [batch][N][SREC_PAD]
  const double *term;  // [batch][TREC]   [Q | q | C | d]
  const double *G0;    // [batch][nc0*nx] column-major
  const double *g0;    // [batch][nc0]
  // backward outputs
  double *ff;   // [batch][N][NR]          [k; z; a]
  double *fb;   // [batch][N][NR*NX]       row-major [K; Z; Ahat]
  double *Vxx;  // [batch][N+1][NX*NX]     column-major (packed-Vxx builds: see Vxx0)
  double *vx;   // [batch][N+1][NX]
  double *ffT;  // [batch][nct]            terminal z
  double *fbT;  // [batch][nct*NX]         terminal Z (row-major)
  double *kkt0; // [batch][NX+nc0]         initial-stage solution [x0; lbda0]
  // forward outputs
  double *xs;    // [batch][N+1][NX]
  double *us;    // [batch][N][NU]
  double *vs;    // [batch][N][NC]
  double *vsT;   // [batch][nct]
  double *lbd0;  // [batch][nc0]
  double *lbdas; // [batch][N][NX]         lbda_1..lbda_N
  int *status;   // [batch]
  int *pivstat;  // [batch] or null: bits 0-14 = 2x2 pivots, bit 15 = initial system on the register fast path, high 16 = interchanges
  // launch tuning (device only; 0 = off)
  int stagger_ns;  // start-up delay per resident warp slot: de-phases the warps of an SM
  int num_sms;
  int ctas_per_sm; // host-side launch hint: resident CTAs per SM wanted (0 = whatever fits)
  int stage_head;  // ring head of the stage records: knot t lives in slot (t + stage_head) mod N (O(1) cycleAppend)
  // parametric problems (nth > 0; CTA-per-instance kernel only): riccati-kernel.hxx:185-192, 278-311
  int nth;
  const double *theta; // [batch][nth] or null (forward)
  double *fth;         // [batch][N][NR*nth]      row-major [Kth; Zth; Yth]
  double *Vxt;         // [batch][N+1][NX*nth]    column-major
  double *Vtt;         // [batch][N+1][nth*nth]
  double *vt;          // [batch][N+1][nth]
  double *kkt0fth;     // [batch][(NX+nc0)*nth]   row-major
  double *thGrad;      // [batch][nth]
  double *thHess;      // [batch][nth*nth]
  // leg mode (CTA-per-instance kernel only): gar::ParallelRiccatiSolver, gar/parallel-solver.hxx.
  // legs = T >= 2: the horizon of every instance is cut into T legs [i(N+1)/T, (i+1)(N+1)/T)
  // (:23-28); a work item of the kernel is one (instance, leg).  nth = nx; records are plain.
  int legs;
  long long *clk; // profiling aid (null = off): per-phase clock64() sums of instance 0's CTA, riccati_block.cuh
  double *cond; // [batch][nc0 + nx*(2T-1)]: condensed solution [lbda0, x0, (theta_i, x_{head i+1})...] (:92-112)
  // Sharded batch: the one exchange of the path (first-step policy [K0 | k0] of every instance, SURVEY 8e) fused
  // into the sweep.  As soon as an instance's backward pass reaches knot 0 its group stores the 
  // nu x (nx+1) block straight into EVERY rank's receive buffer (NVLink peer memory; posted stores that
  // overlap the rest of the sweep).  peer_world = 0: off.  Warp-per-instance kernels only.
  // No flag is awaited inside the sweep (a persistent kernel that spins on something another kernel of the same
  // GPU must produce can starve that kernel of an SM slot): the host side orders this launch after the peers'
  // acknowledgements (ab2_gar_policy_allgather of the previous step).
  int peer_world;
  double *peer_dst[8]; // receive buffer of rank w (peer-mapped)
  long long peer_off;  // doubles: slot * world * batch * per + rank * batch * per
  // Packed-Vxx builds (Cfg::VXX_PACKED, vxx_layout.h): Vxx holds [batch][N+1][vxx_packed_doubles(NX)] and this
  // [batch][NX*NX] array the full block of factor slot 0.  The full-layout build never reads it.
  double *Vxx0;
  // Per-instance mu ([batch], device) of the *_v entry points, or null: every instance uses mueq.  A non-null array
  // selects the kernels' per-instance instantiation (InstanceMu); the programs themselves never read this field.
  const double *mueq_b;
};

// Where a program reads mu: mu(p, inst) at every use.  ScalarMu (the default) is p.mueq, so the scalar launches run
// the programs exactly as they were; InstanceMu is the per-instance array of the *_v launches, read at the use, which
// keeps it out of the registers across the knot loop.
struct ScalarMu {
  AB2_HD double operator()(const SweepParams &p, int) const { return p.mueq; }
};
struct InstanceMu {
  AB2_HD double operator()(const SweepParams &p, int inst) const { return p.mueq_b[inst]; }
};

// status bits: see ST_*; in leg mode several CTAs report on one instance.  ST_BAD_MU: the per-instance mu of a
// *_v backward was not > 0 while constraints are present (set by the kernels, after the program's own status word)
enum : int { ST_CONDENSED_FACTOR_FAILED = 4, ST_BAD_MU = 8 };
// After the backward pass of a per-instance launch (the program has written its status word; `writer` is the thread
// that wrote it): an instance whose mu is unusable -- not > 0, NaN included -- while constraints are present gets
// ST_BAD_MU.  Kernel code only; atomic because several CTAs report on one instance in leg mode.
AB2_D void flag_bad_mu(const SweepParams &p, const int inst, const bool constrained, const bool writer) {
#if defined(__CUDACC__)
  if (p.do_bwd && writer && constrained && !(p.mueq_b[inst] > 0.0))
    atomicOr(p.status + inst, (int)ST_BAD_MU);
#endif
}

// physical slot of stage knot t in the (ring-indexed) stage-record array
AB2_HD int stage_slot(const SweepParams &p, int t) { return ring_slot(t, p.stage_head, p.N); }
// leg i of T over a horizon of N stage knots + the terminal knot (get_work, parallel-solver.hxx:23-28)
AB2_HD int leg_begin(int N, int i, int T) { return (int)((long long)i * (N + 1) / T); }
// doubles before block b of the condensed vector: blocks [nc0, nx, nx, nx, ...]
AB2_HD int cond_offset(int b, int nc0, int nx) { return b == 0 ? 0 : nc0 + (b - 1) * nx; }

// ---------------------------------------------------------------------------
// Compile-time shape of one kernel instantiation.
// ---------------------------------------------------------------------------
template <int NX_, int NU_, int NC_, int G_, bool DB_ = false, bool RB_ = true, bool MMA_ = false, bool PK_ = false>
struct Cfg {
  static constexpr int NX = NX_, NU = NU_, NC = NC_, G = G_;
  static constexpr bool DB = DB_;          // double-buffered knot records
  // Vxx stored as packed lower triangles + a full slot-0 array (vxx_layout.h); false: [N+1][NX*NX] blocks
  static constexpr bool VXX_PACKED = PK_;
  static constexpr int VP = vxx_packed_doubles(NX);
  static constexpr int VXX_REC = PK_ ? VP : NX * NX; // doubles per knot of p.Vxx
  static constexpr int NCOL = NX + NU + 1; // columns of M = [A | B | f]
  static constexpr int NXU = NX + NU;      // rows of H
  static constexpr int NK = NU + NC;       // reduced KKT size
  static constexpr int NR = NU + NC + NX;  // rows of ff / fb
  static constexpr int FCOL = NX + NU;     // the lane that owns f / q,r / ff
  static constexpr bool EVEN = (NX % 2) == 0; // 16-byte aligned rows -> 128-bit LDS
  static constexpr bool REGBK = RB_ && (NU_ + NC_ <= 8); // Bunch-Kaufman entirely in registers
  // unconstrained knots: branch-free register fast path, general algorithm as fallback
  static constexpr bool FASTBK = RB_ && NC_ == 0 && NU_ <= 8;
  static constexpr int ev(int x) { return (x + 1) & ~1; }
  // ---- tensor-core (DMMA m8n8k4) formulation of the stage step ----
  // logical column order [A | f | B] (state, affine, control); tiles of 8 (rows/cols)
  // and 4 (contraction).
  static constexpr bool MMA = MMA_;
  static constexpr int MTX = (NX + 7) / 8;      // m-tiles over state rows
  static constexpr int KT = (NX + 3) / 4;       // k-tiles over the state dimension
  static constexpr int NJ = NX + 1 + NU;        // logical columns
  static constexpr int NT = (NJ + 7) / 8;       // tiles over logical rows/columns of H
  static constexpr int NT2 = (NX + 1 + 7) / 8;  // tiles over [state | affine] columns
  static constexpr int KT2 = (NU + NC + 3) / 4; // k-tiles over the KKT dimension
  // smallest stride >= n that is 4 or 12 mod 16 (conflict-free 64-bit fragment loads)
  static constexpr int fstride(int n) {
    int s = n;
    while (s % 16 != 4 && s % 16 != 12)
      ++s;
    return s;
  }
  static constexpr int VS = MMA ? fstride(4 * KT) : NX;   // row stride of V' in smem
  static constexpr int VROWS = MMA ? 8 * MTX : NX;
  static constexpr int SW = MMA ? ((8 * NT) % 16 == 8 ? 8 * NT : 8 * NT + 8) : 0; // W row stride (== 8 mod 16)
  static constexpr int WROWS = MMA ? 4 * KT : 0;
  static constexpr int SX = MMA ? fstride(8 * NT2) : 0;  // row stride of X / KK
  static constexpr int XROWS = MMA ? 4 * KT2 : 0;
  // [Qhat | qhat] waits in V''s storage during the factorisation and the solves (frees 16 registers where the
  // pressure peaks).  Pays where the double-buffered build spills; the single-buffer build of wider shapes
  // has the registers and would only pay the round trip through shared memory.
  static constexpr bool PARK = MMA_ && DB_;
  // packed Vxx_t store of the tensor-core step: lane l writes the packed pairs l, l + 32, ...
  static constexpr int VPU = (PK_ && MMA_) ? (VP / 2 + 31) / 32 : 0;
  static constexpr int LUT_INTS = MMA ? 32 * (NT + NT * NT + VPU) : 0; // per-CTA table of per-lane constants
  // stage record offsets (doubles), lq_record.cuh
  static constexpr StageOffsets REC = stage_offsets(NX, NU, NC);
  static constexpr int OFF_A = REC.A, OFF_B = REC.B, OFF_F = REC.f, OFF_Q = REC.Q, OFF_S = REC.S, OFF_R = REC.R;
  static constexpr int OFF_QV = REC.q, OFF_RV = REC.r, OFF_C = REC.C, OFF_D = REC.D, OFF_DV = REC.d;
  static constexpr int SREC = REC.end;
  static constexpr int SREC_PAD = stage_pad(SREC); // 16-byte granularity for bulk copies
  static constexpr int M_DBL = OFF_Q;        // [A|B|f]
  static constexpr int SPLIT = ev(M_DBL);    // part 0 = [0,SPLIT), part 1 = rest
  static constexpr int RS = ev(NX + 1);      // row stride of rhs0 / sol
  // shared-memory layout of one group (doubles); every region starts 16-byte aligned
  static constexpr int S_REC = 0;
  // tensor-core step: two zero doubles behind each record buffer -- the entry every
  // structural zero of H0 points at (no compare/select when the accumulators are loaded)
  static constexpr int RSTRIDE = SREC_PAD + (MMA ? 2 : 0);
  static constexpr int S_VN = S_REC + (DB ? 2 : 1) * RSTRIDE; // V' (symmetric, full)
  static constexpr int S_VXN = S_VN + ev(VROWS * VS);          // vx'
  static constexpr int S_KKT = S_VXN + ev(NX);                 // NK*NK column-major
  static constexpr int S_RHS = S_KKT + ev(NK * NK);            // NK x RS, unsolved rhs
  static constexpr int S_SOL = S_RHS + (MMA ? 0 : NK * RS); // (the tensor-core step keeps these in X / KK)
  static constexpr int S_DD = S_SOL + (MMA ? 0 : NK * RS);
  static constexpr int S_SD = S_DD + ev(NK);
  static constexpr int S_X = S_SD + ev(NK);    // forward state x_t (NX) + x_{t+1} (NX)
  static constexpr int S_INT = S_X + 2 * ev(NX); // perm[NK], kind[NK] (ints)
  // MMA staging: W = V' M (WROWS x SW) is dead once H is formed, so it shares its storage
  // with X (control rows of H, XROWS x SX) and KK ([K k; Z z], XROWS x SX).
  static constexpr int S_WSM = S_INT + ev(NK + 1);
  static constexpr int S_XM = S_WSM;
  static constexpr int S_KK = S_XM + ev(XROWS * SX);
  static constexpr int S_MMA_END = S_WSM + (ev(WROWS * SW) > 2 * ev(XROWS * SX) ? ev(WROWS * SW) : 2 * ev(XROWS * SX));
  static constexpr int S_STAGE_END = S_MMA_END;
  static_assert(!MMA || SREC_PAD < 0xffff, "record offsets are packed in 16 bits");
  static_assert(!MMA || (G_ == 32 && NC_ == 0 && (NX_ % 2 == 0)),
                "the tensor-core step needs a full warp, nc = 0, even nx");

  // rec offset of logical column jp of [A | f | B] (padding columns alias column 0)
  static AB2_HD int col_offset(int jp) {
    if (jp < NX)
      return jp * NX;
    if (jp == NX)
      return OFF_F;
    if (jp <= NX + NU)
      return OFF_B + (jp - NX - 1) * NX;
    return 0;
  }
  // rec offset of H0[ip][jp] in logical order, H0 = [[Q q S],[.. 0 ..],[S^T r R]]; -1 = zero
  static AB2_HD int h0_offset(int ip, int jp) {
    const int ti = ip < NX ? 0 : (ip == NX ? 1 : (ip <= NX + NU ? 2 : 3));
    const int tj = jp < NX ? 0 : (jp == NX ? 1 : (jp <= NX + NU ? 2 : 3));
    const int ci = ip - NX - 1, cj = jp - NX - 1;
    if (ti == 0 && tj == 0)
      return OFF_Q + jp * NX + ip;
    if (ti == 0 && tj == 2)
      return OFF_S + cj * NX + ip;
    if (ti == 2 && tj == 0)
      return OFF_S + ci * NX + jp;
    if (ti == 2 && tj == 2)
      return OFF_R + cj * NU + ci;
    if (ti == 0 && tj == 1)
      return OFF_QV + ip;
    if (ti == 2 && tj == 1)
      return OFF_RV + ci;
    return -1;
  }

  // forward rollout: slots of the fb ring (as many as the stage area can hold, at most 8)
  static constexpr bool FB_BULK = ((NR * NX) % 2) == 0; // 16-byte granularity for bulk copies
  // Fused forward: the ring slot of knot t also carries Vxx_t and vx_t
  // -- laid out behind the gain rows as NX more "rows" plus their bias -- so the lanes that
  // pass 1 leaves idle compute lbda_t = vx_t + Vxx_t x_t in the same iteration: no second
  // pass, no register-staged global loads.
  // (only when the lambda rows find idle lanes: nu + nc + 2 nx <= G)
  static constexpr bool FWD_FUSED = FB_BULK && (NX % 2 == 0) && (NR + NX <= G);
  static constexpr int FWD_ROWS = FWD_FUSED ? NR + NX : NR;
  static constexpr bool FWD_FF = FWD_FUSED && (NR % 2 == 0); // ff_t rides in the slot too (no LDG in pass 1)
  // fused slot: [K; Z; Ahat]_t (NR*NX) | Vxx_t (VXX_REC) | vx_t (NX) | ff_t (NR, FWD_FF)
  static constexpr int FWD_BIAS = NR * NX + VXX_REC;
  static constexpr int FWD_SLOT = FWD_FUSED ? FWD_BIAS + NX + (FWD_FF ? NR : 0) : ev(NR * NX); // doubles per ring slot
  static constexpr int FWD_RING_RAW = (S_STAGE_END - 2 * ev(NX)) / FWD_SLOT;
  // the fused ring may outgrow the stage area up to 4 slots.  No more: with packed Vxx a 5th slot
  // would grow the C2 tensor-core build by 2.5 % and cost it its 8th resident CTA per SM.
  static constexpr int FWD_RING_MIN = FWD_FUSED ? 4 : 1;
  static constexpr int FWD_RING = FWD_RING_RAW > 8 ? 8 : (FWD_RING_RAW < FWD_RING_MIN ? FWD_RING_MIN : FWD_RING_RAW);
  static constexpr int NXE = ev(NX);
  static constexpr int FWD_END = FWD_RING * FWD_SLOT + 2 * ev(NX);
  static_assert(NU >= 1, "stage knots need nu >= 1");
  static_assert(NCOL <= G, "lane-per-column mapping needs nx+nu+1 <= G");
  static_assert(NK <= G, "cooperative Bunch-Kaufman needs nu+nc <= G");
  static_assert(G == 8 || G == 16 || G == 32, "group size");

  // doubles of shared memory per group for a run with nc0 initial rows
  static AB2_HD int group_doubles(int nc0) {
    const int n0 = NX + nc0;
    const int k0 = n0 * n0 + 6 * n0 + 2; // K0, b, x, dd, sd, out, 2*n0 ints
    int m = S_STAGE_END > k0 ? S_STAGE_END : k0;
    m = m > FWD_END ? m : FWD_END;
    return (m + 1) & ~1;
  }
  static AB2_HD int term_rec(int nct) { return NX * NX + NX + nct * NX + nct; }
};

// 128-bit shared-memory load of two consecutive doubles (p 16-byte aligned).
struct D2 {
  double x, y;
};
AB2_D D2 lds2(const double *p) {
#if defined(__CUDA_ARCH__)
  const double2 v = *reinterpret_cast<const double2 *>(p);
  return D2{v.x, v.y};
#else
  return D2{p[0], p[1]};
#endif
}
// 128-bit global load of two consecutive doubles (p 16-byte aligned).
AB2_D D2 ldg2(const double *p) {
#if defined(__CUDA_ARCH__)
  const double2 v = *reinterpret_cast<const double2 *>(p);
  return D2{v.x, v.y};
#else
  return D2{p[0], p[1]};
#endif
}
// v[0..N) = p[0..N)  (global memory; ALIGNED: p 16-byte aligned and N even)
template <int N, bool ALIGNED> AB2_D void load_row(const double *p, double (&v)[N]) {
  if constexpr (ALIGNED && (N % 2 == 0)) {
    AB2_UNROLL
    for (int k = 0; k < N; k += 2) {
      const D2 a = ldg2(p + k);
      v[k] = a.x;
      v[k + 1 < N ? k + 1 : k] = a.y;
    }
  } else {
    AB2_UNROLL
    for (int k = 0; k < N; ++k)
      v[k] = p[k];
  }
}
// acc + sum_k row[k] * v[k]; `row` is read by the whole group at the same address
// (broadcast).  ALIGNED: row is 16-byte aligned -> LDS.128.
template <int N, bool ALIGNED> AB2_D double dot_bcast(const double *row, const double (&v)[N], double acc) {
  if constexpr (ALIGNED) {
    AB2_UNROLL
    for (int k = 0; k + 1 < N; k += 2) {
      const D2 a = lds2(row + k);
      acc += a.x * v[k];
      acc += a.y * v[k + 1];
    }
    if constexpr (N % 2)
      acc += row[N - 1] * v[N - 1];
  } else {
    AB2_UNROLL
    for (int k = 0; k < N; ++k)
      acc += row[k] * v[k];
  }
  return acc;
}

// ---------------------------------------------------------------------------
// Cooperative Bunch-Kaufman (lower), n <= G, matrix in shared memory.
// Same pivot logic and arithmetic as bunch_kaufman_in_place_unblocked
// (core/bunchkaufman.hpp:46-151), restructured: lane i owns row i; row
// interchanges are applied to whole rows at once (so the "apply to previous
// columns" pass of :406-417 is not needed); D^-1 is kept in dd/sd.
//   kind[k] = 0: 1x1 pivot, 1: first row of a 2x2 pivot, 2: second row.
//   perm[i]  = original index now at position i  (the composed interchanges).
// Returns false where the reference reports NumericalIssue (:58-59).
// ---------------------------------------------------------------------------
// CHUNK > 1: the trailing-row updates fetch CHUNK operand pairs before storing any result
// (the stores to the row would otherwise serialise the loop on possible aliasing); used by
// the CTA-per-instance kernel, whose matrices are large.
template <int CHUNK = 1, class Ctx>
AB2_D bool bk_factor_group(Ctx &ctx, double *a, const int lda, const int n,
                            double *dd, double *sd, int *perm, int *kind, int &pv) {
  const double alpha = 0.6403882032022076; // (1+sqrt(17))/8
  const int lane = ctx.lane;
#define A_(i, j) a[(i) + (j) * lda]
  if (lane < n)
    perm[lane] = lane;
  ctx.sync();
  bool ok = true;
  int k = 0;
  while (k < n) {
    // ---- pivot search: every lane does it redundantly (broadcast reads) ----
    const double akk = A_(k, k);
    const double abs_akk = fabs(akk);
    int imax = k + 1;
    double colmax = 0.0, cval = 0.0;
    if constexpr (CHUNK > 1) { // fetch CHUNK entries, then run the compare chain on registers
      for (int i0 = k + 1; i0 < n; i0 += CHUNK) {
        double v[CHUNK];
        AB2_UNROLL
        for (int u = 0; u < CHUNK; ++u)
          v[u] = A_((i0 + u < n) ? i0 + u : n - 1, k);
        AB2_UNROLL
        for (int u = 0; u < CHUNK; ++u)
          if (i0 + u < n && fabs(v[u]) > colmax) {
            colmax = fabs(v[u]);
            cval = v[u];
            imax = i0 + u;
          }
      }
    } else {
      for (int i = k + 1; i < n; ++i) {
        const double v = A_(i, k);
        if (fabs(v) > colmax) {
          colmax = fabs(v);
          cval = v;
          imax = i;
        }
      }
    }
    if (fmax(abs_akk, colmax) == 0.0) { // singular column: flag, neutral fill
      ok = false;
      ctx.sync();
      if (lane >= k && lane < n) {
        dd[lane] = 0.0;
        sd[lane] = 0.0;
        kind[lane] = 0;
        for (int j = k; j < lane; ++j)
          A_(lane, j) = 0.0;
      }
      break;
    }
    int kp = k, kstep = 1;
    double aii = akk;
    if (!(abs_akk >= colmax * alpha)) {
      double rowmax = 0.0;
      for (int j = k; j < imax; ++j)
        rowmax = fmax(rowmax, fabs(A_(imax, j)));
      for (int i = imax + 1; i < n; ++i)
        rowmax = fmax(rowmax, fabs(A_(i, imax)));
      aii = A_(imax, imax);
      if (abs_akk >= (alpha * colmax) * (colmax / rowmax)) {
        kp = k;
      } else if (fabs(aii) >= alpha * rowmax) {
        kp = imax;
      } else {
        kp = imax;
        kstep = 2;
      }
    }
    const int kk = k + kstep - 1;
    pv += (kstep == 2 ? 1 : 0) + (kp != kk ? 0x10000 : 0); // pivot statistics (ab2_gar_pivot_stats)
    if (kp != kk) { // ---- symmetric interchange kk <-> kp, whole rows ----
      ctx.sync();   // everyone finished reading before anyone writes
      const int i = lane;
      if (i < n) {
        if (i > kp) {
          const double t = A_(i, kk);
          A_(i, kk) = A_(i, kp);
          A_(i, kp) = t;
        } else if (i > kk && i < kp) {
          const double t = A_(i, kk);
          A_(i, kk) = A_(kp, i);
          A_(kp, i) = t;
        } else if (i < k) {
          const double t = A_(kk, i);
          A_(kk, i) = A_(kp, i);
          A_(kp, i) = t;
        } else if (i == kk) {
          const double t = A_(kk, kk);
          A_(kk, kk) = A_(kp, kp);
          A_(kp, kp) = t;
          const int tp = perm[kk];
          perm[kk] = perm[kp];
          perm[kp] = tp;
        }
        if (kstep == 2 && i == k) { // column k of the 2x2 block: rows k+1 <-> kp
          const double t = A_(k + 1, k);
          A_(k + 1, k) = A_(kp, k);
          A_(kp, k) = t;
        }
      }
    }
    ctx.sync(); // S1
    if (kstep == 1) {
      // post-interchange pivot is akk (no swap) or aii (swap with imax)
      const double d11 = 1.0 / ((kp == k) ? akk : aii);
      double xi = 0.0;
      if (lane > k && lane < n) {
        xi = A_(lane, k);
        A_(lane, k) = xi * d11;
      }
      if (lane == k) {
        dd[k] = d11;
        sd[k] = 0.0;
        kind[k] = 0;
      }
      ctx.sync(); // S2
      if (lane > k && lane < n) {
        if constexpr (CHUNK > 1) {
          for (int j0 = k + 1; j0 <= lane; j0 += CHUNK) {
            double l[CHUNK], r[CHUNK];
            AB2_UNROLL
            for (int u = 0; u < CHUNK; ++u) {
              const int j = (j0 + u <= lane) ? j0 + u : lane;
              l[u] = A_(j, k);
              r[u] = A_(lane, j);
            }
            AB2_UNROLL
            for (int u = 0; u < CHUNK; ++u)
              if (j0 + u <= lane)
                A_(lane, j0 + u) = r[u] - l[u] * xi;
          }
        } else {
          for (int j = k + 1; j <= lane; ++j)
            A_(lane, j) -= A_(j, k) * xi;
        }
      }
    } else {
      // 2x2 pivot on (k, k+1): a11 = akk, a22 = aii, a21 = the column-k entry
      // that was at row imax (cval); identical whether or not rows moved.
      const double d21_abs = fabs(cval);
      const double d21_inv = 1.0 / d21_abs;
      const double d11 = d21_inv * aii;
      const double d22 = d21_inv * akk;
      const double t = 1.0 / ((d11 * d22) - 1.0);
      const double d = t * d21_inv;
      const double d21 = cval * d21_inv;
      double x0 = 0.0, x1 = 0.0;
      if (lane > k + 1 && lane < n) {
        x0 = A_(lane, k);
        x1 = A_(lane, k + 1);
        const double wk = ((x0 * d11) - (x1 * d21)) * d;
        const double wkp1 = ((x1 * d22) - (x0 * d21)) * d;
        A_(lane, k) = wk;
        A_(lane, k + 1) = wkp1;
      }
      if (lane == k) {
        dd[k] = d11 * d;
        sd[k] = -d21 * d;
        dd[k + 1] = d22 * d;
        sd[k + 1] = 0.0;
        kind[k] = 1;
        kind[k + 1] = 2;
        A_(k + 1, k) = 0.0;
      }
      ctx.sync(); // S2
      if (lane > k + 1 && lane < n) {
        if constexpr (CHUNK > 1) {
          for (int j0 = k + 2; j0 <= lane; j0 += CHUNK) {
            double l0[CHUNK], l1[CHUNK], r[CHUNK];
            AB2_UNROLL
            for (int u = 0; u < CHUNK; ++u) {
              const int j = (j0 + u <= lane) ? j0 + u : lane;
              l0[u] = A_(j, k);
              l1[u] = A_(j, k + 1);
              r[u] = A_(lane, j);
            }
            AB2_UNROLL
            for (int u = 0; u < CHUNK; ++u)
              if (j0 + u <= lane)
                A_(lane, j0 + u) = r[u] - (x0 * l0[u] + x1 * l1[u]);
          }
        } else {
          for (int j = k + 2; j <= lane; ++j)
            A_(lane, j) -= x0 * A_(j, k) + x1 * A_(j, k + 1);
        }
      }
    }
    ctx.sync(); // S3: trailing block complete before the next search
    k += kstep;
  }
  ctx.sync();
#undef A_
  return ok;
}

// Per-lane solve of one right-hand-side column (n = NK compile-time, x in
// registers).  Same sequence as bunch_kaufman_solve_in_place
// (core/bunchkaufman.hpp:451-518): interchanges, unit-lower solve, D^-1,
// unit-upper solve, inverse interchanges.  F supplies the factor: F.L(i,c),
// F.dd(k), F.sd(k), F.kind(k), F.perm(i) -- from shared memory (broadcast reads)
// or from registers.
template <int NK, class F>
AB2_D void bk_solve_column(const F &f, const double *rhs, double *sol, const int stride,
                           double (&x)[NK]) {
  AB2_UNROLL
  for (int i = 0; i < NK; ++i)
    x[i] = rhs[f.perm(i) * stride];
  AB2_UNROLL
  for (int c = 0; c < NK; ++c) {
    AB2_UNROLL
    for (int i = c + 1; i < NK; ++i)
      x[i] -= f.L(i, c) * x[c];
  }
  AB2_UNROLL
  for (int k = 0; k < NK; ++k) {
    const int kd = f.kind(k);
    const int k1 = (k + 1 < NK) ? k + 1 : k;
    if (kd == 0) {
      x[k] *= f.dd(k);
    } else if (kd == 1 && k + 1 < NK) {
      const double xk = x[k], xk1 = x[k1];
      const double sdk = f.sd(k);
      x[k] = xk * f.dd(k) + xk1 * sdk;
      x[k1] = xk1 * f.dd(k1) + xk * sdk;
    }
  }
  AB2_UNROLL
  for (int c = NK - 1; c >= 0; --c) {
    AB2_UNROLL
    for (int i = c + 1; i < NK; ++i)
      x[c] -= f.L(i, c) * x[i];
  }
  AB2_UNROLL
  for (int i = 0; i < NK; ++i)
    sol[f.perm(i) * stride] = x[i];
  AB2_UNROLL
  for (int i = 0; i < NK; ++i)
    x[i] = sol[i * stride];
}

template <int NK> struct SmemFactor { // factor left in shared memory by bk_factor_group
  const double *a, *d, *s;
  const int *pm, *kd;
  AB2_D double L(int i, int c) const { return a[i + c * NK]; }
  AB2_D double dd(int k) const { return d[k]; }
  AB2_D double sd(int k) const { return s[k]; }
  AB2_D int kind(int k) const { return kd[k]; }
  AB2_D int perm(int i) const { return pm[i]; }
};

// Fast path of the Bunch-Kaufman factorisation for the common case in which every
// pivot test of bunch_kaufman_in_place_unblocked picks the 1x1 pivot without an
// interchange (|a_kk| >= alpha * colmax, core/bunchkaufman.hpp:61; always-true in
// practice for the SPD matrices Rhat = R + B^T V B of unconstrained knots).  Straight
// line code, no branches: it performs exactly the arithmetic of the general algorithm
// on that path and reports whether the assumption held; if it did not, the caller
// discards this result and runs the general algorithm on the untouched matrix.
// Reciprocal for the pivots of the branch-free fast path: hardware seed (MUFU.RCP64H,
// 2^-20 relative error) + two Newton steps -> within an ulp of 1/x, a third of the
// instructions and two thirds of the latency of the IEEE division sequence.
AB2_D double rcp_fast(double x) {
#if defined(__CUDA_ARCH__)
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
  double e = fma(-x, r, 1.0);
  r = fma(r, e, r);
  e = fma(-x, r, 1.0);
  r = fma(r, e, r);
  return r;
#else
  return 1.0 / x;
#endif
}

template <int N> struct FastFactor {
  double a[N][N]; // lower triangle in, L (strictly lower) out
  double d[N];    // inverted pivots
  AB2_D double L(int i, int c) const { return a[i][c]; }
  AB2_D bool factor() {
    const double alpha = 0.6403882032022076; // (1+sqrt(17))/8
    bool good = true;
    AB2_UNROLL
    for (int k = 0; k < N; ++k) {
      const double akk = a[k][k];
      const double abs_akk = fabs(akk);
      // |akk| >= alpha * colmax  <=>  |akk| >= alpha * |a_ik| for every i (rounding is
      // monotone), and a zero pivot fails one of the two tests of the general algorithm
      // either way: one multiply + one compare per entry instead of an fp64 max
      // (which costs a compare and two selects).
      good = good && (abs_akk > 0.0);
      AB2_UNROLL
      for (int i = k + 1; i < N; ++i)
        good = good && (fabs(a[i][k]) * alpha <= abs_akk);
      const double d11 = rcp_fast(akk);
      d[k] = d11;
      AB2_UNROLL
      for (int j = k + 1; j < N; ++j) {
        const double d11xj = a[j][k] * d11;
        AB2_UNROLL
        for (int i = j; i < N; ++i)
          a[i][j] -= d11xj * a[i][k];
      }
      AB2_UNROLL
      for (int i = k + 1; i < N; ++i)
        a[i][k] *= d11;
    }
    return good;
  }
  // solve with identity interchanges and 1x1 pivots (bunchkaufman.hpp:451-518 on that path)
  AB2_D void solve(const double *rhs, const int stride, double (&x)[N]) const {
    AB2_UNROLL
    for (int i = 0; i < N; ++i)
      x[i] = rhs[i * stride];
    AB2_UNROLL
    for (int c = 0; c < N; ++c) {
      AB2_UNROLL
      for (int i = c + 1; i < N; ++i)
        x[i] -= a[i][c] * x[c];
    }
    AB2_UNROLL
    for (int k = 0; k < N; ++k)
      x[k] *= d[k];
    AB2_UNROLL
    for (int c = N - 1; c >= 0; --c) {
      AB2_UNROLL
      for (int i = c + 1; i < N; ++i)
        x[c] -= a[i][c] * x[i];
    }
  }
};

// Bunch-Kaufman of an N x N matrix held in registers by EVERY lane of the group:
// all lanes run the same scalar algorithm on the same data, so there is no shared
// memory traffic, no synchronisation and no divergence inside a group.  Identical
// pivot logic / arithmetic to bunch_kaufman_in_place_unblocked
// (core/bunchkaufman.hpp:46-151); the dynamic pivot row is resolved by fully
// unrolled compare chains so every register index is static.
template <int N> struct RegFactor {
  double a[N][N]; // lower triangle: L below the diagonal after factor()
  double d[N], s[N];
  int pm[N], kd[N];
  AB2_D double L(int i, int c) const { return a[i][c]; }
  AB2_D double dd(int k) const { return d[k]; }
  AB2_D double sd(int k) const { return s[k]; }
  AB2_D int kind(int k) const { return kd[k]; }
  AB2_D int perm(int i) const { return pm[i]; }

  // symmetric interchange KK <-> C (static), rows swapped across ALL columns
  // K0 = first column of the current pivot block.
  AB2_D void swap_sym(const int KK, const int C, const int K0, const bool two) {
    AB2_UNROLL
    for (int i = 0; i < N; ++i) {
      if (i > C) {
        const double t = a[i][KK];
        a[i][KK] = a[i][C];
        a[i][C] = t;
      } else if (i > KK && i < C) {
        const double t = a[i][KK];
        a[i][KK] = a[C][i];
        a[C][i] = t;
      } else if (i < K0) {
        const double t = a[KK][i];
        a[KK][i] = a[C][i];
        a[C][i] = t;
      }
    }
    {
      const double t = a[KK][KK];
      a[KK][KK] = a[C][C];
      a[C][C] = t;
      const int tp = pm[KK];
      pm[KK] = pm[C];
      pm[C] = tp;
    }
    if (two) { // column K0 of the 2x2 block: rows K0+1 (= KK) <-> C
      const double t = a[KK][K0];
      a[KK][K0] = a[C][K0];
      a[C][K0] = t;
    }
  }

  // one elimination step with a COMPILE-TIME column index (so that every register
  // index stays static even if the compiler declines to unroll a large loop body)
  template <int K> AB2_D void step(bool &ok, bool &skip, bool &dead, int &pv) {
    constexpr int k = K;
    const double alpha = 0.6403882032022076; // (1+sqrt(17))/8
    if (skip || dead) {
      skip = false;
      return;
    }
    const double akk = a[k][k];
    const double abs_akk = fabs(akk);
    int imax = k + 1;
    double colmax = 0.0;
    AB2_UNROLL
    for (int i = k + 1; i < N; ++i) {
      const double v = fabs(a[i][k]);
      if (v > colmax) {
        colmax = v;
        imax = i;
      }
    }
    if (fmax(abs_akk, colmax) == 0.0) {
      ok = false;
      dead = true;
      AB2_UNROLL
      for (int i = k; i < N; ++i) {
        AB2_UNROLL
        for (int j = k; j < i; ++j)
          a[i][j] = 0.0;
      }
      return;
    }
    int kp = k, kstep = 1;
    if (!(abs_akk >= colmax * alpha)) {
      double rowmax = 0.0, aii = akk;
      AB2_UNROLL
      for (int c = k + 1; c < N; ++c)
        if (imax == c) {
          AB2_UNROLL
          for (int j = k; j < c; ++j)
            rowmax = fmax(rowmax, fabs(a[c][j]));
          AB2_UNROLL
          for (int i = c + 1; i < N; ++i)
            rowmax = fmax(rowmax, fabs(a[i][c]));
          aii = a[c][c];
        }
      if (abs_akk >= (alpha * colmax) * (colmax / rowmax)) {
        kp = k;
      } else if (fabs(aii) >= alpha * rowmax) {
        kp = imax;
      } else {
        kp = imax;
        kstep = 2;
      }
    }
    constexpr int k1 = (k + 1 < N) ? k + 1 : k;
    pv += (kstep == 2 ? 1 : 0) + (kp != k + kstep - 1 ? 0x10000 : 0); // pivot statistics
    if (kstep == 1) {
      if (kp != k) {
        AB2_UNROLL
        for (int c = k + 1; c < N; ++c)
          if (kp == c)
            swap_sym(k, c, k, false);
      }
      const double d11 = 1.0 / a[k][k];
      d[k] = d11;
      AB2_UNROLL
      for (int j = k + 1; j < N; ++j) {
        const double d11xj = a[j][k] * d11;
        AB2_UNROLL
        for (int i = j; i < N; ++i)
          a[i][j] -= d11xj * a[i][k];
      }
      AB2_UNROLL
      for (int i = k + 1; i < N; ++i)
        a[i][k] *= d11;
    } else if (k + 1 < N) {
      if (kp != k1) {
        AB2_UNROLL
        for (int c = k + 2; c < N; ++c)
          if (kp == c)
            swap_sym(k1, c, k, true);
      }
      const double d21v = a[k1][k];
      const double d21_abs = fabs(d21v);
      const double d21_inv = 1.0 / d21_abs;
      const double d11 = d21_inv * a[k1][k1];
      const double d22 = d21_inv * a[k][k];
      const double t = 1.0 / ((d11 * d22) - 1.0);
      const double dm = t * d21_inv;
      const double d21 = d21v * d21_inv;
      d[k] = d11 * dm;
      s[k] = -d21 * dm;
      d[k1] = d22 * dm;
      kd[k] = 1;
      kd[k1] = 2;
      AB2_UNROLL
      for (int j = k + 2; j < N; ++j) {
        const double wk = ((a[j][k] * d11) - (a[j][k1] * d21)) * dm;
        const double wkp1 = ((a[j][k1] * d22) - (a[j][k] * d21)) * dm;
        AB2_UNROLL
        for (int i = j; i < N; ++i)
          a[i][j] -= a[i][k] * wk + a[i][k1] * wkp1;
        a[j][k] = wk;
        a[j][k1] = wkp1;
      }
      a[k1][k] = 0.0;
      skip = true;
    }
  }
  template <int... Ks>
  AB2_D void steps(bool &ok, bool &skip, bool &dead, int &pv, std::integer_sequence<int, Ks...>) {
    (step<Ks>(ok, skip, dead, pv), ...);
  }

  AB2_D bool factor(int &pv) {
    bool ok = true, skip = false, dead = false;
    AB2_UNROLL
    for (int i = 0; i < N; ++i) {
      pm[i] = i;
      kd[i] = 0;
      d[i] = 0.0;
      s[i] = 0.0;
    }
    steps(ok, skip, dead, pv, std::make_integer_sequence<int, N>{});
    return ok;
  }
};

// Group-cooperative solve of ONE vector (runtime n <= G): lane i owns x[i].
// b: input (n), x: work/output in permuted order, out: un-permuted result.
template <class Ctx>
AB2_D void bk_solve_vec_group(Ctx &ctx, const double *a, const int lda, const int n,
                               const double *dd, const double *sd, const int *perm,
                               const int *kind, const double *b, double *x, double *out) {
  const int lane = ctx.lane;
  if (lane < n)
    x[lane] = b[perm[lane]];
  for (int c = 0; c < n; ++c) { // column-oriented unit-lower solve
    ctx.sync();
    const double xc = x[c];
    if (lane > c && lane < n)
      x[lane] -= a[lane + c * lda] * xc;
  }
  ctx.sync();
  if (lane < n) {
    const int kd = kind[lane];
    if (kd == 0) {
      x[lane] *= dd[lane];
    } else if (kd == 1) {
      const double xk = x[lane], xk1 = x[lane + 1];
      const double s = sd[lane];
      x[lane] = xk * dd[lane] + xk1 * s;
      x[lane + 1] = xk1 * dd[lane + 1] + xk * s;
    }
  }
  for (int i = n - 1; i >= 1; --i) { // unit-upper solve with L^T
    ctx.sync();
    const double xi = x[i];
    if (lane < i)
      x[lane] -= a[i + lane * lda] * xi;
  }
  ctx.sync();
  if (lane < n)
    out[perm[lane]] = x[lane];
  ctx.sync();
}


// ---------------------------------------------------------------------------
// Fast path of the initial saddle system [[Vxx_0, G0^T],[G0, 0]] x = b
// (proximal-riccati.hxx:44-55): LDL^T for the case in which every pivot test of the
// Bunch-Kaufman algorithm picks the 1x1 pivot in place by its first test
// (|a_kk| >= alpha*colmax, core/bunchkaufman.hpp:61) -- what happens for the saddle systems
// of well-posed problems.  Same arithmetic, in the same order, as bk_factor_group +
// bk_solve_vec_group on that path (so the result is identical), but: lane = row, the column
// test is a vote instead of a redundant scan by every lane, the pivot column's entries
// travel by shuffles, every shared-memory access is conflict-free (odd leading dimension),
// the solves keep x in a register.  About a tenth of the general routine's shared-memory
// wavefronts.  Returns false at the first failing test with the matrix partly overwritten:
// the caller then rebuilds it and runs the general algorithm.
//   a: n x n, lower triangle, column-major with ODD leading dimension lda.
template <class Ctx>
AB2_D bool kkt0_fast(Ctx &ctx, double *a, const int lda, const int n, const double rhs, double &x_out) {
  const double alpha = 0.6403882032022076; // (1+sqrt(17))/8
  const int lane = ctx.lane;
  const bool in = lane < n;
  double myd = 0.0;
  for (int k = 0; k < n; ++k) {
    ctx.sync(); // column k is final
    const double akk = a[k + k * lda];
    const bool below = lane > k && in;
    const double my = below ? a[lane + k * lda] : 0.0;
    const bool ok = (fabs(my) * alpha <= fabs(akk)) && (fabs(akk) > 0.0);
    if (!ctx.all(ok))
      return false;
    const double d = 1.0 / akk;
    if (lane == k)
      myd = d;
    // trailing rows: a_ij -= (a_jk d) a_ik, i >= j > k; four columns per round so that the
    // shuffles and loads of a round are in flight together
    int j = k + 1;
    for (; j + 4 <= n; j += 4) {
      const double m0 = ctx.shfl(my, j), m1 = ctx.shfl(my, j + 1), m2 = ctx.shfl(my, j + 2),
                   m3 = ctx.shfl(my, j + 3);
      double *pj = a + (in ? lane : 0) + j * lda;
      const double r0 = pj[0], r1 = pj[lda], r2 = pj[2 * lda], r3 = pj[3 * lda];
      if (in && lane >= j)
        pj[0] = r0 - (m0 * d) * my;
      if (in && lane >= j + 1)
        pj[lda] = r1 - (m1 * d) * my;
      if (in && lane >= j + 2)
        pj[2 * lda] = r2 - (m2 * d) * my;
      if (in && lane >= j + 3)
        pj[3 * lda] = r3 - (m3 * d) * my;
    }
    for (; j < n; ++j) {
      const double mj = ctx.shfl(my, j);
      if (in && lane >= j)
        a[lane + j * lda] -= (mj * d) * my;
    }
    if (below)
      a[lane + k * lda] = my * d;
  }
  ctx.sync();
  double x = rhs;
  for (int c = 0; c + 1 < n; ++c) { // unit-lower solve, column-oriented (bunchkaufman.hpp:472)
    const double xc = ctx.shfl(x, c);
    if (lane > c && in)
      x -= a[lane + c * lda] * xc;
  }
  x *= myd; // D^-1 (1x1 pivots, :499)
  for (int i = n - 1; i >= 1; --i) { // unit-upper solve with L^T (:504)
    const double xi = ctx.shfl(x, i);
    if (lane < i)
      x -= a[i + lane * lda] * xi;
  }
  x_out = x;
  ctx.sync(); // everyone is done with the matrix
  return true;
}

// 128-bit global store of two consecutive doubles (p 16-byte aligned).
AB2_D void stg2(double *p, double x, double y) {
#if defined(__CUDA_ARCH__)
  *reinterpret_cast<double2 *>(p) = make_double2(x, y);
#else
  p[0] = x;
  p[1] = y;
#endif
}

// 128-bit shared-memory store of two consecutive doubles (p 16-byte aligned).
AB2_D void sts2(double *p, double x, double y) {
#if defined(__CUDA_ARCH__)
  *reinterpret_cast<double2 *>(p) = make_double2(x, y);
#else
  p[0] = x;
  p[1] = y;
#endif
}

// Per-CTA table of per-lane constants of the tensor-core step: lut[t][lane] = record offset of
// logical column 8t+g; lut[NT + mt*NT + nt][lane] = packed record offsets of the two H0
// entries of accumulator tile (mt, nt) (structural zeros point at the zero slot behind the
// record).  Written by ONE warp of the CTA (or one host thread per lane) before any sweep.
template <class C> AB2_HD void fill_mma_lut(int *lut, const int lane, const int first = 0, const int step = 1) {
  constexpr int NT = C::NT;
  const int g = lane >> 2, q = lane & 3;
  for (int r = first; r < NT + NT * NT; r += step) { // table rows are dealt out over the CTA's warps
    if (r < NT) {
      lut[r * 32 + lane] = C::col_offset(8 * r + g);
    } else {
      const int mt = (r - NT) / NT, nt = (r - NT) % NT;
      const int o0 = C::h0_offset(8 * mt + g, 8 * nt + 2 * q);
      const int o1 = C::h0_offset(8 * mt + g, 8 * nt + 2 * q + 1);
      const unsigned u0 = o0 < 0 ? (unsigned)C::SREC_PAD : (unsigned)o0; // structural zero -> the zero slot
      const unsigned u1 = o1 < 0 ? (unsigned)C::SREC_PAD : (unsigned)o1;
      lut[r * 32 + lane] = (int)(u0 | (u1 << 16));
    }
  }
  // packed Vxx_t store: offsets in V' of the two entries of packed pair (r - NT - NT*NT) * 32 + lane,
  // row j of V' for entry (i, j) (contiguous along a packed column); 0xffff = the zero padding entry
  for (int r = NT + NT * NT + first; r < NT + NT * NT + C::VPU; r += step) {
    const int e0 = 2 * ((r - NT - NT * NT) * 32 + lane);
    unsigned u[2];
    for (int e = 0; e < 2; ++e) {
      u[e] = 0xffffu;
      if (e0 + e < C::NX * (C::NX + 1) / 2) {
        int i, j;
        vxx_packed_coords(C::NX, e0 + e, i, j);
        u[e] = (unsigned)(j * C::VS + i);
      }
    }
    lut[r * 32 + lane] = (int)(u[0] | (u[1] << 16));
  }
}

// ---------------------------------------------------------------------------
// Stage knots N-1..0 on the FP64 tensor cores (mma.sync m8n8k4, SASS DMMA).
//
// Same mathematics as the lane-per-column loop below (riccati-kernel.hxx:210-277);
// the four dense products are tiled 8x8x4 and issued as DMMAs, whose operands live
// in registers: shared memory is touched once per FRAGMENT instead of once per FMA
// (the lane-per-column form needs one broadcast shared-memory operand per DFMA and
// saturates the LSU pipe, while one DMMA does 8x8x4 FMAs from four register operands).
// Logical column order [A | f | B]; with lane = 4 g + q:
//   A fragment (8x4):  lane holds a[g][q]          B fragment (4x8): lane holds b[q][g]
//   C/D fragment (8x8): lane holds d[g][2q], d[g][2q+1]
//  (1) W  = V' M                MTX x NT tiles, KT k-steps   (A: V' from smem, B: M from rec)
//  (2) H  = H0 + M^T W          NT  x NT tiles, KT k-steps   (A: the SAME M fragments, B: W via smem)
//  (3) control rows of H -> X (right-hand sides) and the KKT matrix; Bunch-Kaufman + solves
//  (4) [Ahat a] = [A f] + B KK  MTX x NT2 tiles, KT2 k-steps (A: B from rec, B: KK via smem)
//  (5) [Vxx vx] = [Qhat qhat] + X^T KK            same shapes (A: X from smem, B: same KK)
// ---------------------------------------------------------------------------
template <class C, class Ctx>
AB2_D void stage_loop_mma(Ctx &ctx, const SweepParams &p, double *__restrict__ sm, int &st, int &pv,
                          const int inst) {
  constexpr int NX = C::NX, NU = C::NU, NK = C::NK, NR = C::NR;
  constexpr int MTX = C::MTX, KT = C::KT, NT = C::NT, NT2 = C::NT2, KT2 = C::KT2;
  constexpr int VS = C::VS, SW = C::SW, SX = C::SX;
  const int lane = ctx.lane;
  const int g = lane >> 2, q = lane & 3;
  const int N = p.N;
  // Output / input bases are re-derived from the kernel parameters (constant bank) where
  // they are used instead of being carried in registers across the whole loop.
#define AB2_STAGE_B (p.stage + (size_t)inst * N * C::SREC_PAD)
#define AB2_FF_B (p.ff + (size_t)inst * N * NR)
#define AB2_FB_B (p.fb + (size_t)inst * N * NR * NX)
#define AB2_VXX_B (p.Vxx + (size_t)inst * (N + 1) * C::VXX_REC)
#define AB2_VXX0_B (C::VXX_PACKED ? p.Vxx0 + (size_t)inst * NX * NX : AB2_VXX_B)
#define AB2_VX_B (p.vx + (size_t)inst * (N + 1) * NX)
  double *Vn = sm + C::S_VN;
  double *vxn = sm + C::S_VXN;
  double *kkt = sm + C::S_KKT;
  double *dd = sm + C::S_DD;
  double *sd = sm + C::S_SD;
  int *perm = reinterpret_cast<int *>(sm + C::S_INT);
  int *kind = perm + NK;
  double *Wsm = sm + C::S_WSM;
  double *X = sm + C::S_XM;
  double *KKs = sm + C::S_KK;

  // per-lane constants: record offsets of the logical columns 8t+g and of H0's entries.
  // They live in a small per-CTA table in shared memory, filled ONCE per CTA before the
  // sweeps start (fill_mma_lut, called by the kernel prologue), instead of 12 registers
  // that would be spilled to local memory, which has no L1 behind it in this kernel.
  const int *lut = ctx.cta_ints(); // [(NT + NT*NT)][32]
  if (lane < (C::DB ? 4 : 2))
    sm[C::S_REC + (lane >> 1) * C::RSTRIDE + C::SREC_PAD + (lane & 1)] = 0.0;
  for (int i = lane; i < C::S_MMA_END - C::S_WSM; i += 32)
    Wsm[i] = 0.0; // W / X / KK share this space; its padding entries must be finite
  ctx.sync();

  const bool colS = lane <= NX; // this lane solves right-hand-side column `lane` ([K | k])
  int cur = 0;
  for (int t = N - 1; t >= 0; --t) {
    // DB: the record of knot t-1 streams into the other buffer during this step.
    // Single buffer (smaller footprint -> more resident CTAs): the record is refilled in two
    // parts as soon as each is consumed -- the cost blocks after (2), [A|B|f] after (5).
    ctx.wait_copy(C::DB ? cur : 0);
    double *rec = sm + C::S_REC + (C::DB ? cur : 0) * C::RSTRIDE;
    if (C::DB) {
      if (t > 0)
        ctx.issue_copy(cur ^ 1, sm + C::S_REC + (cur ^ 1) * C::RSTRIDE,
                       AB2_STAGE_B + (size_t)stage_slot(p, t - 1) * C::SREC_PAD, C::SREC_PAD);
      cur ^= 1;
    }

    // fragments of M = [A | f | B]: B-operand of (1) and A-operand (M^T) of (2)
    double Mf[NT][KT];
    AB2_UNROLL
    for (int tt = 0; tt < NT; ++tt) {
      AB2_UNROLL
      for (int kt = 0; kt < KT; ++kt)
        Mf[tt][kt] = rec[lut[tt * 32 + lane] + 4 * kt + q];
    }
    // (1) W = V' M   (+ vx' on the affine column: vplus = vx' + V' f, :217-218)
    {
      double W[MTX][NT][2];
      AB2_UNROLL
      for (int mt = 0; mt < MTX; ++mt) {
        AB2_UNROLL
        for (int nt = 0; nt < NT; ++nt) {
          W[mt][nt][0] = 0.0;
          W[mt][nt][1] = 0.0;
        }
      }
      AB2_UNROLL
      for (int kt = 0; kt < KT; ++kt) { // contraction outermost: MTX*NT independent DMMAs per step
        AB2_UNROLL
        for (int mt = 0; mt < MTX; ++mt) {
          const double va = Vn[(8 * mt + g) * VS + 4 * kt + q];
          AB2_UNROLL
          for (int nt = 0; nt < NT; ++nt)
            ctx.mma(W[mt][nt], va, Mf[nt][kt]);
        }
      }
      AB2_UNROLL
      for (int mt = 0; mt < MTX; ++mt) {
        const int i = 8 * mt + g;
        if (i < NX) {
          AB2_UNROLL
          for (int nt = 0; nt < NT; ++nt) {
            AB2_UNROLL
            for (int e = 0; e < 2; ++e)
              if (8 * nt + 2 * q + e == NX)
                W[mt][nt][e] += vxn[i];
            sts2(Wsm + i * SW + 8 * nt + 2 * q, W[mt][nt][0], W[mt][nt][1]);
          }
        }
      }
    }
    ctx.sync();
    // (2) H = H0 + M^T W
    if (!C::DB)
      ctx.wait_copy(1); // the cost blocks of this knot
    double H[NT][NT][2];
    AB2_UNROLL
    for (int mt = 0; mt < NT; ++mt) {
      AB2_UNROLL
      for (int nt = 0; nt < NT; ++nt) {
        AB2_UNROLL
        for (int e = 0; e < 2; ++e) {
          const unsigned o = ((unsigned)lut[(NT + mt * NT + nt) * 32 + lane] >> (16 * e)) & 0xffffu;
          H[mt][nt][e] = rec[o];
        }
      }
    }
    AB2_UNROLL
    for (int kt = 0; kt < KT; ++kt) {
      AB2_UNROLL
      for (int nt = 0; nt < NT; ++nt) {
        // rows >= NX pad the contraction (never stored): structural zeros
        const double wb = (4 * kt + q < NX) ? Wsm[(4 * kt + q < NX ? 4 * kt + q : 0) * SW + 8 * nt + g] : 0.0;
        AB2_UNROLL
        for (int mt = 0; mt < NT; ++mt)
          ctx.mma(H[mt][nt], Mf[mt][kt], wb);
      }
    }
    // (3) control rows of H: [Shat^T | rhat] -> X, Rhat -> KKT matrix (:232-257)
    ctx.sync(); // every lane has its W fragments: the storage becomes X / KK
    if (!C::DB && t > 0) // ... and its H0 entries: the cost blocks of knot t-1 may land
      ctx.issue_copy(1, rec + C::SPLIT, AB2_STAGE_B + (size_t)stage_slot(p, t - 1) * C::SREC_PAD + C::SPLIT,
                     C::SREC_PAD - C::SPLIT);
    AB2_UNROLL
    for (int mt = 0; mt < NT; ++mt) {
      const int c = 8 * mt + g - NX - 1;
      if (c >= 0 && c < NU) {
        AB2_UNROLL
        for (int nt = 0; nt < NT; ++nt) {
          AB2_UNROLL
          for (int e = 0; e < 2; ++e) {
            const int jp = 8 * nt + 2 * q + e;
            if (jp <= NX)
              X[c * SX + jp] = H[mt][nt][e];
            else if (jp - NX - 1 < NU)
              kkt[c + (jp - NX - 1) * NK] = H[mt][nt][e]; // Rhat[c][c2]
          }
        }
      }
    }
    // The state rows of H ([Qhat | qhat], the initial value of the accumulators of (5)) wait in
    // shared memory while the factorisation and the solves run: V' and vx' are dead since (1),
    // their storage is exactly the right shape, and 16 registers are free when the register
    // pressure peaks (the spills this avoids went to local memory, which has no L1 behind it here).
    if (C::PARK) {
      AB2_UNROLL
      for (int mt = 0; mt < MTX; ++mt) {
        const int i = 8 * mt + g;
        if (i < NX) {
          AB2_UNROLL
          for (int nt = 0; nt < NT2; ++nt) {
            const int j0 = 8 * nt + 2 * q;
            if (j0 + 1 < NX)
              sts2(Vn + i * VS + j0, H[mt][nt][0], H[mt][nt][1]);
            else if (j0 == NX)
              vxn[i] = H[mt][nt][0];
          }
        }
      }
    }
    ctx.sync();
    double *fbt = AB2_FB_B + (size_t)t * NR * NX;
    double *fft = AB2_FF_B + (size_t)t * NR;
    {
      double kz[NK];
      FastFactor<NK> F;
      AB2_UNROLL
      for (int c = 0; c < NK; ++c) {
        AB2_UNROLL
        for (int i = c; i < NK; ++i)
          F.a[i][c] = kkt[i + c * NK];
      }
      if (F.factor()) { // uniform over the warp
        if (colS)
          F.solve(X + lane, SX, kz);
      } else { // an interchange / 2x2 pivot / singular column: general algorithm
        if (!bk_factor_group(ctx, kkt, NK, NK, dd, sd, perm, kind, pv))
          st |= ST_STAGE_FACTOR_FAILED;
        if (colS) {
          const SmemFactor<NK> G{kkt, dd, sd, perm, kind};
          bk_solve_column<NK>(G, X + lane, KKs + lane, SX, kz); // KKs doubles as scratch
        }
      }
      if (colS) { // the right-hand side is -X: negate the solution; outputs K / k
        double *const odst = (lane < NX) ? fbt + lane : fft;
        const int ostride = (lane < NX) ? NX : 1;
        AB2_UNROLL
        for (int c = 0; c < NK; ++c) {
          const double v = -kz[c];
          KKs[c * SX + lane] = v;
          odst[c * ostride] = v;
        }
      }
    }
    ctx.sync();
    // fragments of KK = [K k].  No predicates: rows >= NK meet the structural zeros of the
    // other operand (they only have to be finite -- the buffer was zeroed once and is
    // shared with W), columns > NX feed accumulator entries nobody stores.
    double KKf[KT2][NT2];
    AB2_UNROLL
    for (int k2 = 0; k2 < KT2; ++k2) {
      AB2_UNROLL
      for (int nt = 0; nt < NT2; ++nt)
        KKf[k2][nt] = KKs[(4 * k2 + q) * SX + 8 * nt + g];
    }
    // (4) [Ahat a] = [A f] + B KK   (:266-267)   and
    // (5) [Vxx vx] = [Qhat qhat] + Shat KK, with Shat[i][c] = X[c][i]   (:270-277)
    // All operand fragments are fetched first and the two products are interleaved with the
    // contraction outermost: 2*MTX*NT2 independent DMMAs per k-step.
    {
      double EA[MTX][NT2][2], VV[MTX][NT2][2], Bf[MTX][KT2], Xf[MTX][KT2];
      AB2_UNROLL
      for (int mt = 0; mt < MTX; ++mt) { // [Qhat | qhat] back from where it waited (entries nobody stores: any finite value)
        const int i = 8 * mt + g;
        const int ic2 = i < NX ? i : 0;
        AB2_UNROLL
        for (int nt = 0; nt < NT2; ++nt) {
          const int j0 = 8 * nt + 2 * q;
          if (!C::PARK) {
            VV[mt][nt][0] = H[mt][nt][0];
            VV[mt][nt][1] = H[mt][nt][1];
          } else if (j0 + 1 < NX) {
            const D2 v = lds2(Vn + ic2 * VS + j0);
            VV[mt][nt][0] = v.x;
            VV[mt][nt][1] = v.y;
          } else {
            VV[mt][nt][0] = vxn[ic2];
            VV[mt][nt][1] = 0.0;
          }
        }
      }
      AB2_UNROLL
      for (int mt = 0; mt < MTX; ++mt) {
        const int i = 8 * mt + g;
        const int ic = i < NX ? i : 0;
        AB2_UNROLL
        for (int nt = 0; nt < NT2; ++nt) {
          AB2_UNROLL
          for (int e = 0; e < 2; ++e) {
            // rows i >= NX and columns jj > NX of the accumulator are never stored: any
            // finite value will do there, so no select
            const int jj = 8 * nt + 2 * q + e;
            const int off = (jj < NX) ? jj * NX : ((jj == NX) ? C::OFF_F : 0);
            EA[mt][nt][e] = rec[off + ic];
          }
        }
        AB2_UNROLL
        for (int k2 = 0; k2 < KT2; ++k2) {
          const int c = 4 * k2 + q;
          // (rows i >= NX of both accumulators are never stored: no row predicate)
          const double bv = rec[C::OFF_B + (c < NU ? c : 0) * NX + ic];
          Bf[mt][k2] = (c < NU) ? bv : 0.0;
          const double xv = X[c * SX + i];
          Xf[mt][k2] = (c < NK) ? xv : 0.0;
        }
      }
      AB2_UNROLL
      for (int k2 = 0; k2 < KT2; ++k2) {
        AB2_UNROLL
        for (int mt = 0; mt < MTX; ++mt) {
          AB2_UNROLL
          for (int nt = 0; nt < NT2; ++nt) {
            ctx.mma(EA[mt][nt], Bf[mt][k2], KKf[k2][nt]);
            ctx.mma(VV[mt][nt], Xf[mt][k2], KKf[k2][nt]);
          }
        }
      }
      if (!C::DB && t > 0) {
        // single buffer: [A|B|f] of this knot now lives in the accumulators and fragments of every
        // lane (the products above consumed the loads): refill it while the results are stored
        ctx.sync();
        ctx.issue_copy(0, rec, AB2_STAGE_B + (size_t)stage_slot(p, t - 1) * C::SREC_PAD, C::SPLIT);
      }
      AB2_UNROLL
      for (int mt = 0; mt < MTX; ++mt) {
        const int i = 8 * mt + g;
        if (i < NX) {
          AB2_UNROLL
          for (int nt = 0; nt < NT2; ++nt) {
            AB2_UNROLL
            for (int e = 0; e < 2; ++e) {
              const int jj = 8 * nt + 2 * q + e;
              if (jj < NX)
                fbt[(NK + i) * NX + jj] = EA[mt][nt][e];
              else if (jj == NX)
                fft[NK + i] = EA[mt][nt][e];
            }
          }
        }
      }
      AB2_UNROLL
      for (int mt = 0; mt < MTX; ++mt) {
        const int i = 8 * mt + g;
        if (i < NX) {
          AB2_UNROLL
          for (int nt = 0; nt < NT2; ++nt) {
            AB2_UNROLL
            for (int e = 0; e < 2; ++e) {
              const int jj = 8 * nt + 2 * q + e;
              const double v = VV[mt][nt][e];
              if (jj < NX) {
                if (t == 0)
                  AB2_VXX0_B[i + jj * NX] = v; // datas[0].Vxx is left unsymmetrised (A1)
                if (i >= jj) {            // V' = lower triangle mirrored (:216 of the next step)
                  Vn[i * VS + jj] = v;
                  Vn[jj * VS + i] = v;
                }
              } else if (jj == NX) {
                AB2_VX_B[(size_t)t * NX + i] = v;
                vxn[i] = v;
              }
            }
          }
        }
      }
    }
    ctx.sync();
    if (t > 0) { // symmetric Vxx_t, as the next step of the reference leaves it
      double *Vt = AB2_VXX_B + (size_t)t * C::VXX_REC;
      if constexpr (C::VXX_PACKED) { // the lower triangle, packed: one 16-byte store per pair of entries
        AB2_UNROLL
        for (int u = 0; u < C::VPU; ++u) {
          const int e = 2 * (u * 32 + lane);
          if (e < C::VP) {
            const unsigned o = (unsigned)lut[(NT + NT * NT + u) * 32 + lane];
            const unsigned o0 = o & 0xffffu, o1 = o >> 16;
            stg2(Vt + e, o0 == 0xffffu ? 0.0 : Vn[o0], o1 == 0xffffu ? 0.0 : Vn[o1]);
          }
        }
      } else if (lane < NX) { // row `lane` of the symmetric V' = column `lane` of Vxx_t
        if (C::EVEN && (VS % 2 == 0)) {
          AB2_UNROLL
          for (int i = 0; i < NX; i += 2) {
            const D2 v = lds2(Vn + lane * VS + i);
            stg2(Vt + i + lane * NX, v.x, v.y);
          }
        } else {
          AB2_UNROLL
          for (int i = 0; i < NX; ++i)
            Vt[i + lane * NX] = Vn[lane * VS + i];
        }
      }
    }
  }
}
#undef AB2_STAGE_B
#undef AB2_FF_B
#undef AB2_FB_B
#undef AB2_VXX_B
#undef AB2_VXX0_B
#undef AB2_VX_B

// Lane j < NX stores packed column j (rows j..NX-1) of the symmetric V' (row j of V' in shared memory);
// lane 0 also writes the padding entry.
template <class C> AB2_D void store_packed_column(double *dst, const double *Vn, const int lane) {
  constexpr int NX = C::NX;
  double *col = dst + vxx_packed_col(NX, lane) - lane; // col[i] = entry (i, lane)
  AB2_UNROLL
  for (int i = 0; i < NX; ++i)
    if (i >= lane)
      col[i] = Vn[lane * C::VS + i];
  if (C::VP > NX * (NX + 1) / 2 && lane == 0)
    dst[C::VP - 1] = 0.0;
}

// ---------------------------------------------------------------------------
// The sweep of one instance by one group.
// ---------------------------------------------------------------------------
// mu: where this instance's mu is read (ScalarMu / InstanceMu above).
template <class C, class Ctx, class Mu = ScalarMu>
AB2_D void riccati_group_sweep(Ctx &ctx, const SweepParams &p, const int inst,
                                double *__restrict__ sm, const Mu &mu = Mu()) {
  constexpr int NX = C::NX, NU = C::NU, NC = C::NC, NK = C::NK, NR = C::NR;
  constexpr int NXU = C::NXU, NCOL = C::NCOL, FCOL = C::FCOL;
  const int lane = ctx.lane;
  const int N = p.N;
  const int nct = p.nct, nc0 = p.nc0;

  double *rec = sm + C::S_REC; // current knot record (buffer 0 / alternating when DB)
  double *Vn = sm + C::S_VN;
  double *vxn = sm + C::S_VXN;
  double *kkt = sm + C::S_KKT;
  double *rhs0 = sm + C::S_RHS;
  double *sol = sm + C::S_SOL;
  double *dd = sm + C::S_DD;
  double *sd = sm + C::S_SD;
  double *xv = sm + C::S_X;
  int *perm = reinterpret_cast<int *>(sm + C::S_INT);
  int *kind = perm + NK;

  const double *stage_b = p.stage + (size_t)inst * N * C::SREC_PAD;
  double *ff_b = p.ff + (size_t)inst * N * NR;
  double *fb_b = p.fb + (size_t)inst * N * NR * NX;
  double *Vxx_b = p.Vxx + (size_t)inst * (N + 1) * C::VXX_REC;
  double *Vxx0_b = C::VXX_PACKED ? p.Vxx0 + (size_t)inst * NX * NX : Vxx_b; // the block of slot 0, full
  double *vx_b = p.vx + (size_t)inst * (N + 1) * NX;
  int st = ST_OK;
  int pv = 0; // pivot statistics: +1 per 2x2 pivot, +0x10000 per interchange

  // lane classes
  const bool colA = lane < NX;                 // owns a state column
  const bool colB = lane >= NX && lane < NXU;  // owns a control column
  const bool colF = lane == FCOL;              // owns the affine column
  const bool active = lane < NCOL;
  const int jj = colF ? NX : lane; // column index in rhs0/sol (feedback cols, then ff)

  if (p.do_bwd) {
    // prefetch the last stage knot while the terminal knot is processed
    if (N > 0) {
      const double *src = stage_b + (size_t)stage_slot(p, N - 1) * C::SREC_PAD;
      if (C::DB) {
        ctx.issue_copy(0, rec, src, C::SREC_PAD);
      } else {
        ctx.issue_copy(0, rec, src, C::SPLIT);
        ctx.issue_copy(1, rec + C::SPLIT, src + C::SPLIT, C::SREC_PAD - C::SPLIT);
      }
    }
    if constexpr (C::MMA) { // padded rows/columns of V' must hold zeros (fragment loads read them)
      for (int i = lane; i < C::VROWS * C::VS; i += C::G)
        Vn[i] = 0.0;
      ctx.sync();
    }
    // ---------------- terminal knot (nu = 0): riccati-kernel.hxx:146-149,175-183
    {
      const double *tr = p.term + (size_t)inst * C::term_rec(nct);
      const double *Qt = tr;
      const double *qt = tr + NX * NX;
      const double *Ct = qt + NX;            // nct x NX column-major
      const double *dt = Ct + (size_t)nct * NX;
      double *VN = N > 0 ? Vxx_b + (size_t)N * C::VXX_REC : Vxx0_b;
      if (colA || colF) {
        // column j of Z = C/mu (or z = d/mu), then column j of Q + C^T Z (q + C^T z)
        double acc[NX];
        AB2_UNROLL
        for (int i = 0; i < NX; ++i)
          acc[i] = 0.0;
#if defined(__CUDACC__)
#pragma unroll 1
#endif
        for (int m = 0; m < nct; ++m) {
          const double zm = (colF ? dt[m] : Ct[m + (size_t)lane * nct]) / mu(p, inst);
          if (colF)
            p.ffT[(size_t)inst * nct + m] = zm;
          else
            p.fbT[(size_t)inst * nct * NX + (size_t)m * NX + lane] = zm;
          AB2_UNROLL
          for (int i = 0; i < NX; ++i)
            acc[i] += Ct[m + (size_t)i * nct] * zm;
        }
        AB2_UNROLL
        for (int i = 0; i < NX; ++i) {
          const double s = (colF ? qt[i] : Qt[i + lane * NX]) + acc[i];
          if (colF) {
            vx_b[(size_t)N * NX + i] = s;
            vxn[i] = s;
          } else {
            if (!C::VXX_PACKED || N == 0)
              VN[i + lane * NX] = s; // as computed; re-written symmetric below when N > 0
            if (i >= lane) {       // V' for the next step = lower triangle mirrored (:216)
              Vn[i * C::VS + lane] = s;
              Vn[lane * C::VS + i] = s;
            }
          }
        }
      }
      ctx.sync();
      if (colA && N > 0) { // step N-1 of the reference symmetrises datas[N].Vxx in place (A1)
        if constexpr (C::VXX_PACKED)
          store_packed_column<C>(VN, Vn, lane);
        else {
          AB2_UNROLL
          for (int i = 0; i < NX; ++i)
            VN[i + lane * NX] = Vn[lane * C::VS + i];
        }
      }
    }

    // ---------------- stage knots N-1 .. 0: riccati-kernel.hxx:210-277
    if constexpr (C::MMA) {
      stage_loop_mma<C>(ctx, p, sm, st, pv, inst);
    } else {
    constexpr int RS = C::RS;
    constexpr bool EV = C::EVEN;
    int cur = 0; // record buffer in use (DB)
    for (int t = N - 1; t >= 0; --t) {
      if (C::DB) {
        ctx.wait_copy(cur);
        rec = sm + C::S_REC + cur * C::RSTRIDE;
        if (t > 0) // stream the next knot into the other buffer during this step
          ctx.issue_copy(cur ^ 1, sm + C::S_REC + (cur ^ 1) * C::RSTRIDE,
                         stage_b + (size_t)stage_slot(p, t - 1) * C::SREC_PAD, C::SREC_PAD);
        cur ^= 1;
      } else {
        ctx.wait_copy(0);
        ctx.wait_copy(1);
      }
      // own column of M = [A|B|f]
      double mcol[NX];
      if (EV) {
        AB2_UNROLL
        for (int k = 0; k < NX; k += 2) {
          const D2 v = lds2(rec + (active ? lane : 0) * NX + k);
          mcol[k] = v.x;
          mcol[k + 1 < NX ? k + 1 : k] = v.y;
        }
      } else {
        AB2_UNROLL
        for (int k = 0; k < NX; ++k)
          mcol[k] = rec[(active ? lane : 0) * NX + k];
      }
      // (A) w = V' m_j  (+ vx' on the affine column: vplus = vx' + V' f, :217-218)
      double w[NX];
      AB2_UNROLL
      for (int i = 0; i < NX; ++i)
        w[i] = dot_bcast<NX, EV>(Vn + i * C::VS, mcol, 0.0);
      if (colF) {
        AB2_UNROLL
        for (int i = 0; i < NX; ++i)
          w[i] += vxn[i];
      }
      // (B) H[:,j] = H0[:,j] + [A B]^T w      (:220-228 in one product)
      // H0 = [[Q S q],[S^T R r]]; per-lane base/stride so the code is uniform
      int base1, base2, stride2;
      if (colA) {
        base1 = C::OFF_Q + lane * NX;
        base2 = C::OFF_S + lane;
        stride2 = NX;
      } else if (colB) {
        base1 = C::OFF_S + (lane - NX) * NX;
        base2 = C::OFF_R + (lane - NX) * NU;
        stride2 = 1;
      } else {
        base1 = C::OFF_QV;
        base2 = C::OFF_RV;
        stride2 = 1;
      }
      // control rows first: they go straight to the KKT matrix / right-hand sides
      // (:232-257) and never occupy registers afterwards
      // colB lanes: Rhat[:,c] -> KKT column c (only r >= c is read); colA/colF lanes:
      // -Shat^T[:,j] / -rhat -> right-hand-side column jj.  One predicated store, no branch.
      double *const cdst = colB ? kkt + (lane - NX) * NK : rhs0 + jj;
      const int cstride = colB ? 1 : RS;
      const double csign = colB ? 1.0 : -1.0;
      AB2_UNROLL
      for (int r = 0; r < NU; ++r) {
        const double hr = dot_bcast<NX, EV>(rec + (NX + r) * NX, w, rec[base2 + r * stride2]);
        if (active)
          cdst[r * cstride] = csign * hr;
      }
      if (colB) {
        AB2_UNROLL
        for (int m = 0; m < NC; ++m)
          kkt[NU + m + (lane - NX) * NK] = rec[C::OFF_D + (lane - NX) * NC + m];
      }
      if (lane < NC) { // (1,1) block: -mu on the diagonal, zeros below
        AB2_UNROLL
        for (int m = 0; m < NC; ++m)
          kkt[NU + m + (NU + lane) * NK] = (m == lane) ? -mu(p, inst) : 0.0;
      }
      if (colA || colF) {
        AB2_UNROLL
        for (int m = 0; m < NC; ++m)
          rhs0[(NU + m) * RS + jj] = colF ? -rec[C::OFF_DV + m] : -rec[C::OFF_C + lane * NC + m];
      }
      // state rows: Qhat[:,j] / Shat[:,c] / qhat stay in registers for step (E)
      // With double-buffered records each lane parks its column in the slot it read
      // H0[:,j] from (private to the lane) so it does not occupy registers during the
      // factorisation; the single-buffer variant refills that slot early and keeps it
      // in registers instead.
      constexpr bool STASH = C::DB;
      double h[NX];
      AB2_UNROLL
      for (int i = 0; i < NX; ++i) {
        h[i] = dot_bcast<NX, EV>(rec + i * NX, w, rec[base1 + i]);
        if (STASH && (colA || colF)) // Q column j / q: read by this lane only
          rec[base1 + i] = h[i];
      }
      ctx.sync();
      if (!C::DB && t > 0) // part 1 of the record (Q..d) is consumed: fetch the next knot's
        ctx.issue_copy(1, rec + C::SPLIT, stage_b + (size_t)stage_slot(p, t - 1) * C::SREC_PAD + C::SPLIT,
                       C::SREC_PAD - C::SPLIT);
      // (C) Bunch-Kaufman of the reduced KKT matrix, (D) solve + closed loop (:259-267)
      double kz[NK];
      double *fbt = fb_b + (size_t)t * NR * NX;
      double *fft = ff_b + (size_t)t * NR;
      if constexpr (C::FASTBK) {
        FastFactor<NK> F;
        AB2_UNROLL
        for (int c = 0; c < NK; ++c) {
          AB2_UNROLL
          for (int i = c; i < NK; ++i)
            F.a[i][c] = kkt[i + c * NK];
        }
        if (F.factor()) { // uniform over the group: every lane factored the same matrix
          if (colA || colF)
            F.solve(rhs0 + jj, RS, kz);
        } else { // an interchange / 2x2 pivot / singular column: general algorithm
          if (!bk_factor_group(ctx, kkt, NK, NK, dd, sd, perm, kind, pv))
            st |= ST_STAGE_FACTOR_FAILED;
          if (colA || colF) {
            const SmemFactor<NK> G{kkt, dd, sd, perm, kind};
            bk_solve_column<NK>(G, rhs0 + jj, sol + jj, RS, kz);
          }
        }
      } else if constexpr (C::REGBK) {
        RegFactor<NK> F;
        AB2_UNROLL
        for (int c = 0; c < NK; ++c) {
          AB2_UNROLL
          for (int i = c; i < NK; ++i)
            F.a[i][c] = kkt[i + c * NK];
        }
        if (!F.factor(pv))
          st |= ST_STAGE_FACTOR_FAILED;
        if (colA || colF)
          bk_solve_column<NK>(F, rhs0 + jj, sol + jj, RS, kz);
      } else {
        if (!bk_factor_group(ctx, kkt, NK, NK, dd, sd, perm, kind, pv))
          st |= ST_STAGE_FACTOR_FAILED;
        if (colA || colF) {
          const SmemFactor<NK> F{kkt, dd, sd, perm, kind};
          bk_solve_column<NK>(F, rhs0 + jj, sol + jj, RS, kz);
        }
      }
      if (colA || colF) {
        // [Ahat a] = [A f] + B [K k]
        double ahat[NX];
        AB2_UNROLL
        for (int i = 0; i < NX; ++i)
          ahat[i] = STASH ? rec[lane * NX + i] : mcol[i];
        AB2_UNROLL
        for (int c = 0; c < NU; ++c) {
          const double kc = kz[c];
          if (EV) {
            AB2_UNROLL
            for (int i = 0; i < NX; i += 2) {
              const D2 b = lds2(rec + C::OFF_B + c * NX + i);
              ahat[i] += b.x * kc;
              ahat[i + 1 < NX ? i + 1 : i] += b.y * kc;
            }
          } else {
            AB2_UNROLL
            for (int i = 0; i < NX; ++i)
              ahat[i] += rec[C::OFF_B + c * NX + i] * kc;
          }
        }
        // column `lane` of fb (stride NX) or the vector ff (stride 1): same code
        double *const odst = colA ? fbt + lane : fft;
        const int ostride = colA ? NX : 1;
        AB2_UNROLL
        for (int r = 0; r < NK; ++r)
          odst[r * ostride] = kz[r];
        AB2_UNROLL
        for (int i = 0; i < NX; ++i)
          odst[(NK + i) * ostride] = ahat[i];
      }
      if (!C::DB) {
        ctx.sync();
        if (t > 0) // part 0 ([A|B|f]) is consumed
          ctx.issue_copy(0, rec, stage_b + (size_t)stage_slot(p, t - 1) * C::SREC_PAD, C::SPLIT);
      }
      // (E) cost-to-go: [Vxx vx] = [Qhat qhat] + [Shat C^T][K k; Z z]   (:270-277)
      if (colA || colF) {
        if (STASH) {
          AB2_UNROLL
          for (int i = 0; i < NX; ++i)
            h[i] = rec[base1 + i];
        }
        // rhs0 still holds -Shat^T (rows 0..NU-1) and -C (rows NU..NK-1)
        AB2_UNROLL
        for (int r = 0; r < NU; ++r) {
          const double kr = kz[r];
          if (EV) {
            AB2_UNROLL
            for (int i = 0; i < NX; i += 2) {
              const D2 sv = lds2(rhs0 + r * RS + i);
              h[i] -= sv.x * kr;
              h[i + 1 < NX ? i + 1 : i] -= sv.y * kr;
            }
          } else {
            AB2_UNROLL
            for (int i = 0; i < NX; ++i)
              h[i] -= rhs0[r * RS + i] * kr;
          }
        }
        if (NC > 0) {
          double s2[NX];
          AB2_UNROLL
          for (int i = 0; i < NX; ++i)
            s2[i] = 0.0;
          AB2_UNROLL
          for (int m = 0; m < NC; ++m) {
            const double zr = kz[NU + m < NK ? NU + m : 0];
            AB2_UNROLL
            for (int i = 0; i < NX; ++i)
              s2[i] -= rhs0[(NU + m) * RS + i] * zr;
          }
          AB2_UNROLL
          for (int i = 0; i < NX; ++i)
            h[i] += s2[i];
        }
        if (colA) {
          if (t == 0) { // datas[0].Vxx is left unsymmetrised (A1)
            double *Vt = Vxx0_b;
            AB2_UNROLL
            for (int i = 0; i < NX; ++i)
              Vt[i + lane * NX] = h[i];
          }
          AB2_UNROLL
          for (int i = 0; i < NX; ++i)
            if (i >= lane) { // V' = lower triangle mirrored (:216 of the next step)
              Vn[i * C::VS + lane] = h[i];
              Vn[lane * C::VS + i] = h[i];
            }
        } else {
          AB2_UNROLL
          for (int i = 0; i < NX; ++i) {
            vx_b[(size_t)t * NX + i] = h[i];
            vxn[i] = h[i];
          }
        }
      }
      if (STASH) // the stashed columns were written through the generic proxy into the record
        ctx.proxy_fence_smem(); // buffer the next bulk copy overwrites (issued after the sync below)
      ctx.sync();
      if (t > 0 && colA) { // symmetric Vxx_t, as the next step of the reference leaves it
        double *Vt = Vxx_b + (size_t)t * C::VXX_REC;
        if constexpr (C::VXX_PACKED)
          store_packed_column<C>(Vt, Vn, lane);
        else {
          AB2_UNROLL
          for (int i = 0; i < NX; ++i)
            Vt[i + lane * NX] = Vn[lane * C::VS + i];
        }
      }
    }

    } // lane-per-column stage loop

    // ---------------- sharded batch: this instance's first-step policy goes to every rank now
    if (p.peer_world > 0 && N > 0) {
      ctx.sync(); // the group's own stores of K_0, k_0 are ordered before its loads
      constexpr int PER = NU * (NX + 1);
      const double *fb0 = p.fb + (size_t)inst * N * NR * NX, *ff0 = p.ff + (size_t)inst * N * NR;
      for (int e = lane; e < PER; e += C::G) {
        const int r = e / (NX + 1), c = e - r * (NX + 1);
        const double v = (c < NX) ? fb0[r * NX + c] : ff0[r];
        for (int w = 0; w < p.peer_world; ++w)
          p.peer_dst[w][p.peer_off + (long long)inst * PER + e] = v;
      }
    }

    // ---------------- initial stage: proximal-riccati.hxx:42-55 (nth = 0)
    {
      const int n0 = NX + nc0;
      double *K0 = sm;              // n0 x n0 column-major (overlays the stage area)
      double *b0 = K0 + n0 * n0;
      double *x0w = b0 + n0;
      double *dd0 = x0w + n0;
      double *sd0 = dd0 + n0;
      double *o0 = sd0 + n0;
      int *perm0 = reinterpret_cast<int *>(o0 + n0);
      int *kind0 = perm0 + n0;
      // pull what is needed out of the stage area before overwriting it
      double vcol[NX];
      double vx0 = 0.0;
      AB2_UNROLL
      for (int i = 0; i < NX; ++i)
        vcol[i] = colA ? Vn[i * C::VS + lane] : 0.0;
      if (lane < NX)
        vx0 = vxn[lane];
      ctx.sync();
      const double *G0 = p.G0 + (size_t)inst * nc0 * NX;
      const double *g0 = p.g0 + (size_t)inst * nc0;
      // fast path: LDL^T in registers (lane = column), valid when no pivot test asks for an
      // interchange or a 2x2 pivot; otherwise the general algorithm below, from the same sources
      const int ld0 = n0 | 1; // odd leading dimension: rows and columns both conflict-free
      if (colA) {
        AB2_UNROLL
        for (int i = 0; i < NX; ++i)
          if (i >= lane)
            K0[i + lane * ld0] = vcol[i]; // lower triangle of Vxx_0
        for (int m = 0; m < nc0; ++m)
          K0[NX + m + lane * ld0] = G0[m + (size_t)lane * nc0];
      }
      for (int m = lane; m < nc0; m += C::G)
        for (int m2 = m; m2 < nc0; ++m2)
          K0[NX + m2 + (NX + m) * ld0] = 0.0;
      const double b = (lane < NX) ? -vx0 : ((lane < n0) ? -g0[lane - NX] : 0.0);
      double x = 0.0;
      const bool fast_done = kkt0_fast(ctx, K0, ld0, n0, b, x); // (synchronises before reading)
      if (fast_done && lane < n0)
        p.kkt0[(size_t)inst * n0 + lane] = x;
      if (fast_done)
        pv |= 0x8000; // statistics: the initial system took the fast path
      else
        ctx.sync();   // everyone has left the fast path before the matrix is rebuilt
      if (!fast_done) {
        if (colA) {
          AB2_UNROLL
          for (int i = 0; i < NX; ++i)
            if (i >= lane)
              K0[i + lane * n0] = vcol[i]; // lower triangle of Vxx_0
          for (int m = 0; m < nc0; ++m)
            K0[NX + m + lane * n0] = G0[m + (size_t)lane * nc0];
          b0[lane] = -vx0;
        }
        for (int m = lane; m < nc0; m += C::G) {
          for (int m2 = m; m2 < nc0; ++m2)
            K0[NX + m2 + (NX + m) * n0] = 0.0;
          b0[NX + m] = -g0[m];
        }
        ctx.sync();
        if (!bk_factor_group<4>(ctx, K0, n0, n0, dd0, sd0, perm0, kind0, pv))
          st |= ST_INIT_FACTOR_FAILED;
        bk_solve_vec_group(ctx, K0, n0, n0, dd0, sd0, perm0, kind0, b0, x0w, o0);
        for (int i = lane; i < n0; i += C::G)
          p.kkt0[(size_t)inst * n0 + i] = o0[i];
        ctx.sync();
      }
    }
    if (lane == 0) {
      p.status[inst] = st;
      if (p.pivstat)
        p.pivstat[inst] = pv;
    }
  }

  // ---------------- forward rollout: riccati-kernel.hxx:196-207, 315-377
  if (p.do_fwd) {
    const int n0 = NX + nc0;
    const double *k0 = p.kkt0 + (size_t)inst * n0;
    double *xs_b = p.xs + (size_t)inst * (N + 1) * NX;
    double *us_b = p.us + (size_t)inst * N * NU;
    double *vs_b = p.vs + (size_t)inst * N * NC;
    double *lb_b = p.lbdas + (size_t)inst * N * NX;
    // Pass 1 -- the sequential part: x_{t+1} = a + Ahat x_t (and u, v, which read the same
    // rows of fb).  The fb records stream through a ring of FWD_RING shared-memory slots
    // filled by TMA bulk copies issued FWD_RING knots ahead (no registers, deep enough to
    // cover HBM latency); ff travels in a register pipeline of the same depth.
    constexpr int RING = C::FWD_RING;
    constexpr int FS = C::FWD_SLOT;
    constexpr bool FUSED = C::FWD_FUSED;
    constexpr int ROWS = C::FWD_ROWS;             // gain rows (+ NX lambda rows when fused)
    constexpr int RPL = (ROWS + C::G - 1) / C::G; // rows per lane
    const int NIT = FUSED ? N + 1 : N;            // the fused loop has one more iteration: lbda_N
    constexpr bool EVF = C::EVEN;
    double *ring = sm;                 // RING x FS doubles (the backward's buffers are dead)
    double *xc = sm + RING * FS;       // x_t
    double *xnx = xc + C::NXE;         // x_{t+1}
    (void)xv;
    // The ring's bulk copies overwrite shared memory this group wrote through the generic
    // proxy (initial-stage workspace) and, in the fused sweep, read ff / fb / Vxx / vx this
    // group stored to global memory during the backward pass: every lane orders its
    // generic-proxy writes before the async proxy, then the group synchronises.
    ctx.proxy_fence();
    ctx.sync();
    auto fill_slot = [&](int d, int t) { // fb record of knot t -> ring slot d
      if (FUSED) { // [K; Z; Ahat]_t | Vxx_t (symmetric for t >= 1; no lambda row reads Vxx_0) | vx_t
        constexpr int VR = C::VXX_REC;
        ctx.copy_expect(d, (t < N ? NR * NX + (C::FWD_FF ? NR : 0) : 0) + (t > 0 ? VR : 0) + NX);
        if (t < N) {
          ctx.copy_add(d, ring + d * FS, fb_b + (size_t)t * NR * NX, NR * NX);
          if (C::FWD_FF)
            ctx.copy_add(d, ring + d * FS + C::FWD_BIAS + NX, ff_b + (size_t)t * NR, NR);
        }
        if (t > 0)
          ctx.copy_add(d, ring + d * FS + NR * NX, Vxx_b + (size_t)t * VR, VR);
        ctx.copy_add(d, ring + d * FS + C::FWD_BIAS, vx_b + (size_t)t * NX, NX);
      } else if (C::FB_BULK) {
        ctx.issue_copy(d, ring + d * FS, fb_b + (size_t)t * NR * NX, NR * NX);
      } else { // odd record size: no 16-byte granularity, plain cooperative copy
        for (int i2 = lane; i2 < NR * NX; i2 += C::G)
          ring[d * FS + i2] = fb_b[(size_t)t * NR * NX + i2];
      }
    };
    AB2_UNROLL
    for (int d = 0; d < RING; ++d)
      if (d < NIT)
        fill_slot(d, d);
    if (lane < NX) {
      const double v = k0[lane];
      xc[lane] = v;
      xs_b[lane] = v;
    }
    for (int m = lane; m < nc0; m += C::G)
      p.lbd0[(size_t)inst * nc0 + m] = k0[NX + m];
    double gff[RING][RPL];
    AB2_UNROLL
    for (int d = 0; d < RING; ++d) {
      AB2_UNROLL
      for (int q = 0; q < RPL; ++q) {
        const int r = lane + q * C::G;
        gff[d][q] = (!C::FWD_FF && r < NR && d < N) ? ff_b[(size_t)d * NR + r] : 0.0;
      }
    }
    ctx.sync();
    for (int t0 = 0; t0 < NIT; t0 += RING) {
      AB2_UNROLL
      for (int d = 0; d < RING; ++d) {
        const int t = t0 + d;
        if (t < NIT) {
          if (C::FB_BULK)
            ctx.wait_copy(d);
          const double *slot = ring + d * FS;
          AB2_UNROLL
          for (int q = 0; q < RPL; ++q) {
            const int r = lane + q * C::G;
            // gain rows exist for t < N; lambda rows (fused) for t >= 1
            if (FUSED ? ((r < NR && t < N) || (r >= NR && r < ROWS && t >= 1)) : (r < NR)) {
              double s0 = gff[d][q], s1 = 0.0; // two chains halve the dependent-FMA latency
              if (FUSED && (C::FWD_FF || r >= NR)) // ff_t sits right behind vx_t: one bias vector
                s0 = slot[C::FWD_BIAS + (r >= NR ? r - NR : NX + r)];
              if (EVF) {
                // Row r starts NX/2 16-byte units into the slot: with NX/2 = 2 mod 4 (nx = 4, 12)
                // rows r and r+4 of a quarter-warp's 128-bit load fall on the same banks.  Those
                // rows walk their column pairs rotated by one (pairs 1,2,..,0): the two halves
                // then sit on units of different parity -- no conflict, same products.
                constexpr bool ROT = ((NX / 2) % 4) == 2;
                const int rot2 = ROT ? ((r >> 1) & 2) : 0; // 2 doubles for rows 4..7 (mod 8)
                AB2_UNROLL
                for (int c = 0; c < NX; c += 2) {
                  const int cc = (ROT && c + 2 == NX) ? (rot2 ? 0 : c) : c + rot2;
                  D2 gg;
                  if (C::VXX_PACKED && FUSED && r >= NR) { // row r - NR of the packed symmetric Vxx_t
                    gg.x = slot[NR * NX + vxx_packed_index(NX, r - NR, cc)];
                    gg.y = slot[NR * NX + vxx_packed_index(NX, r - NR, cc + 1)];
                  } else {
                    gg = lds2(slot + r * NX + cc);
                  }
                  const D2 xx = lds2(xc + cc);
                  s0 += gg.x * xx.x;
                  s1 += gg.y * xx.y;
                }
              } else {
                AB2_UNROLL
                for (int c = 0; c < NX; ++c)
                  s0 += slot[r * NX + c] * xc[c];
              }
              const double s = s0 + s1;
              if (r < NU)
                us_b[(size_t)t * NU + r] = s;
              else if (r < NK)
                vs_b[(size_t)t * NC + (r - NU)] = s;
              else if (!FUSED || r < NR) {
                xnx[r - NK] = s;
                xs_b[(size_t)(t + 1) * NX + (r - NK)] = s;
              } else {
                lb_b[(size_t)(t - 1) * NX + (r - NR)] = s; // lbda_t = vx_t + Vxx_t x_t
              }
              if (!C::FWD_FF && (!FUSED || r < NR))
                gff[d][q] = (t + RING < N) ? ff_b[(size_t)(t + RING) * NR + r] : 0.0;
            }
          }
          if (t < N) {
            double *tmp = xc;
            xc = xnx;
            xnx = tmp;
          }
          ctx.sync(); // x_{t+1} visible; every lane is done with x_t and with this slot
          if (t + RING < NIT)
            fill_slot(d, t + RING);
        }
      }
    }
    // Pass 2 -- the parallel part: lbda_{t+1} = vx_{t+1} + Vxx_{t+1} x_{t+1} has no
    // dependence between knots: G/NX knots per iteration, two iterations batched so that
    // all their loads are in flight together; no synchronisation.  A packed row takes one
    // predicated load per entry, and two batched iterations spill at nx = 14: one there.
    if (!FUSED) {
      constexpr int KPI = (C::G / NX) > 0 ? (C::G / NX) : 1; // knots per iteration
      constexpr int U = C::VXX_PACKED ? 1 : 2;
      const int sub = lane / NX, i = lane % NX;
      if (sub < KPI) {
        for (int t = sub; t < N; t += KPI * U) {
          double vrow[U][NX], xr[U][NX], v0[U];
          AB2_UNROLL
          for (int u = 0; u < U; ++u) {
            const int tt = t + u * KPI;
            if (tt < N) {
              if constexpr (C::VXX_PACKED) { // row i of the packed symmetric Vxx_{tt+1}
                // two bases, so that every load has a compile-time offset: entries (c, i), c >= i, lie
                // at lo[c]; entries (i, c), c < i, at up[col(c) - c]
                const double *V = Vxx_b + (size_t)(tt + 1) * C::VXX_REC;
                const double *lo = V + vxx_packed_col(NX, i) - i, *up = V + i;
                AB2_UNROLL
                for (int c = 0; c < NX; ++c) {
                  if (c >= i)
                    vrow[u][c] = lo[c];
                  else
                    vrow[u][c] = up[vxx_packed_col(NX, c) - c];
                }
              } else {
                load_row<NX, EVF>(Vxx_b + ((size_t)(tt + 1) * NX + i) * NX, vrow[u]); // row i (symmetric)
              }
              load_row<NX, EVF>(xs_b + (size_t)(tt + 1) * NX, xr[u]);
              v0[u] = vx_b[(size_t)(tt + 1) * NX + i];
            }
          }
          AB2_UNROLL
          for (int u = 0; u < U; ++u) {
            const int tt = t + u * KPI;
            if (tt < N) {
              double s0 = v0[u], s1 = 0.0;
              AB2_UNROLL
              for (int c = 0; c + 1 < NX; c += 2) {
                s0 += vrow[u][c] * xr[u][c];
                s1 += vrow[u][c + 1] * xr[u][c + 1];
              }
              if (NX % 2)
                s0 += vrow[u][NX - 1] * xr[u][NX - 1];
              lb_b[(size_t)tt * NX + i] = s0 + s1;
            }
          }
        }
      }
      ctx.sync();
    }
    // terminal multipliers v_N = z + Z x_N
    for (int m = lane; m < nct; m += C::G) {
      double s = p.ffT[(size_t)inst * nct + m];
      for (int c = 0; c < NX; ++c)
        s += p.fbT[(size_t)inst * nct * NX + (size_t)m * NX + c] * xc[c];
      p.vsT[(size_t)inst * nct + m] = s;
    }
  }
}

} // namespace ab2
