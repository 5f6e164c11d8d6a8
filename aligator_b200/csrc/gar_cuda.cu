// gar_cuda.cu -- sm_90a kernels + C-ABI implementation (include/aligator_b200/gar.h).
//
// The arithmetic lives in riccati_group.cuh (one group of G lanes per problem
// instance).  This file supplies the device execution context -- TMA bulk copies
// (cp.async.bulk, SASS UBLKCP) completing on per-group mbarriers, or cp.async
// (LDGSTS) staging -- the persistent-sweep kernel, the shape dispatch and the
// host-side handle.  No CPU fallback: every entry point fails loudly without a
// CUDA device.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <string>
#include <utility>
#include <vector>

#include "../../include/aligator_b200/gar.h"
#include "linesearch.h"
#include "lq_adjoint.h"
#include "lq_resolve.h"
#include "lq_theta.h"
#include "lq_factor_adjoint.h"
#include "lq_factor_tangent.h"
#include "lq_jacobian.h"
#include "lq_refine.h"
#include "lq_assemble.h"
#include "proxddp_inner.h"
#include "riccati_block_launch.h"
#include "riccati_configs.h"
#include "riccati_launch.cuh"

namespace ab2 {

// [K_0 | k_0] of every instance -> dst [batch][nu][nx+1]
// (head: physical slot of stage knot 0 in the factor arrays, non-zero only between a cycleAppend and the next backward)
__global__ void first_step_policy_kernel(const double *__restrict__ fb, const double *__restrict__ ff,
                                         double *__restrict__ dst, int batch, int N, int nr, int nu, int nx, int head) {
  const int per = nu * (nx + 1);
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < (long)batch * per; i += (long)gridDim.x * blockDim.x) {
    const int b = (int)(i / per), e = (int)(i % per), r = e / (nx + 1), c = e % (nx + 1);
    const size_t k0 = ((size_t)b * N + head) * nr + r;
    dst[i] = (c < nx) ? fb[k0 * nx + c] : ff[k0];
  }
}

// ---------------------------------------------------------------------------
// Multi-GPU: the all-gather of the first-step policy FUSED into the kernel that computes it, over
// NVLink peer memory.  Every rank owns a receive buffer [3][world][batch][nu][nx+1] (three slots,
// step s lives in slot s mod 3) + flag words, mapped into every peer by CUDA IPC.
//  * warp-per-instance sweeps (SweepParams::peer_*): the sweep kernel itself stores an instance's
//    [K0 | k0] into slot [s mod 3][r] of EVERY rank's buffer the moment its backward pass reaches
//    knot 0 (posted peer stores over NVLink / NVSwitch that overlap the rest of the sweep; no pack
//    kernel, no NCCL kernel, no staging copy); ab2_gar_policy_allgather then only publishes the
//    step number in every peer's data flag (policy_publish_kernel);
//  * every other kernel (CTA per instance, legs, dense): policy_allgather_kernel packs from the
//    factor arrays and stores each element into every rank's slot, the last CTA publishes.
// Flow control: the WAIT kernel of step s (stream-ordered behind the consumers of step s-1 on the
// consumer's stream) first tells every peer "everything up to s-1 is consumed here" (ack flag),
// then waits for the data flags of step s; the publish kernel of step s holds the producer's
// stream until every peer has acknowledged step s-2 -- what the slot of step s+1 held.  A rank may
// thus run two steps ahead of the slowest consumer, and NO flag is ever awaited inside the
// persistent sweep (it would starve the kernel that writes the flag of an SM slot).
// ---------------------------------------------------------------------------
constexpr int kMaxPeers = 8;
struct PeerPtrs {
  double *buf[kMaxPeers];               // receive buffer of rank w
  unsigned long long *data_flag[kMaxPeers]; // [world] of rank w: step of the last block received from each sender
  unsigned long long *ack_flag[kMaxPeers];  // [world] of rank w: last step each peer has finished consuming
};
__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__global__ void __launch_bounds__(256)
    policy_allgather_kernel(const double *__restrict__ fb, const double *__restrict__ ff, const PeerPtrs peers,
                            const int world, const int rank, const int batch, const int N, const int nr, const int nu,
                            const int nx, const unsigned long long step, unsigned int *done_counter) {
  const int per = nu * (nx + 1);
  const long total = (long)batch * per;
  if (threadIdx.x == 0) {
    if (step >= 3) // the slot written now held step-3: every peer has consumed it once it acknowledges step-2
      for (int w = 0; w < world; ++w)
        while (ld_acquire_sys(peers.ack_flag[rank] + w) + 2 < step)
          __nanosleep(64);
  }
  __syncthreads();
  const size_t half = (size_t)(step % 3) * world * total; // three slots
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int b = (int)(i / per), e = (int)(i % per), r = e / (nx + 1), c = e % (nx + 1);
    const double v = (c < nx) ? fb[((size_t)b * N * nr + r) * nx + c] : ff[(size_t)b * N * nr + r];
    for (int w = 0; w < world; ++w) // own buffer first-class: w == rank is a local store
      peers.buf[w][half + (size_t)rank * total + i] = v;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(done_counter, 1u);
    if (prev == gridDim.x - 1) { // every CTA's stores are fenced: publish
      *done_counter = 0;
      __threadfence_system();
      for (int w = 0; w < world; ++w)
        st_release_sys(peers.data_flag[w] + rank, step);
    }
  }
}
// the sweep kernel stored this rank's blocks into every peer itself (SweepParams::peer_*): order them
// before the flags (the kernel boundary orders the sweep's stores before this kernel; the fence and the
// releases carry that to system scope)
// It also holds the stream until every peer has consumed step - 2: the NEXT sweep stores into the slot that held
// step - 2 (three slots).  That wait sits here, in a one-warp kernel behind the sweep, never inside the
// persistent sweep: a kernel that fills every SM and spins on a flag which another kernel of the same GPU must
// write (this rank's own wait kernel, on the side stream) can starve that kernel of an SM slot for ever.
__global__ void policy_publish_kernel(const PeerPtrs peers, const int world, const int rank, const unsigned long long step) {
  const int w = threadIdx.x;
  __threadfence_system();
  if (w < world) {
    st_release_sys(peers.data_flag[w] + rank, step);
    if (step >= 3)
      while (ld_acquire_sys(peers.ack_flag[rank] + w) + 2 < step)
        __nanosleep(64);
  }
}
// the stream waits until the blocks of every sender have arrived for `step`; before that it
// acknowledges to every peer that this rank is done with step-1 (everything enqueued earlier on
// this stream -- the consumers of step-1 -- has completed)
__global__ void policy_wait_kernel(const PeerPtrs peers, const int world, const int rank, const unsigned long long step) {
  const int w = threadIdx.x;
  if (w < world) {
    st_release_sys(peers.ack_flag[w] + rank, step - 1);
    while (ld_acquire_sys(peers.data_flag[rank] + w) < step)
      __nanosleep(64);
  }
}

// row-major fb [nr][nx] + ff [nr]  ->  column-major [nr][nx+1] with column 0 = ff, per (instance, knot)
__global__ void gains_kernel(const double *__restrict__ fb, const double *__restrict__ ff, double *__restrict__ dst,
                             long nrec, int nr, int nx, int N, int head) {
  const int per = nr * (nx + 1);
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < nrec * per; i += (long)gridDim.x * blockDim.x) {
    long rec = i / per; // logical (instance, knot) -> physical slot
    if (head) {
      const long b = rec / N;
      const int t = (int)(rec % N) + head;
      rec = b * N + (t >= N ? t - N : t);
    }
    const int e = (int)(i % per), c = e / nr, r = e % nr; // destination is column-major
    dst[i] = (c == 0) ? ff[rec * nr + r] : fb[(rec * nr + r) * nx + (c - 1)];
  }
}

// ---- FDDP backwardPass bookkeeping around the sweep (solver-fddp.hxx:204-277) ----
// before: slack_t = fs[t+1] (the knot's affine term), G0 = -I, g0 = fs[0]
__global__ void fddp_prep_kernel(const double *__restrict__ fs, double *__restrict__ slack, double *__restrict__ G0,
                                 double *__restrict__ g0, int batch, int N, int nx) {
  const long nS = (long)batch * N * nx, nG = (long)batch * nx * nx, ng = (long)batch * nx;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < nS + nG + ng; i += (long)gridDim.x * blockDim.x) {
    if (i < nS) {
      const long b = i / ((long)N * nx), r = i % ((long)N * nx);
      slack[i] = fs[b * (N + 1) * nx + nx + r];
    } else if (i < nS + nG) {
      const long e = (i - nS) % ((long)nx * nx);
      G0[i - nS] = (e % nx == e / nx) ? -1.0 : 0.0;
    } else {
      const long j = i - nS - nG, b = j / nx, c = j % nx;
      g0[j] = fs[b * (N + 1) * nx + c];
    }
  }
}
// after: Vx_i = vx_i + sym(Vxx_i) fs[i] (:219-220, 272-276), then Quuks_i = -(Lu_i + Ju_i^T Vx_{i+1}) = Quu_i k_i (:264)
// (Vxx0 != null: Vxx in the packed layout of vxx_layout.h, knot t in factor slot t)
__global__ void fddp_vx_kernel(const double *__restrict__ Vxx, const double *__restrict__ Vxx0, const double *__restrict__ vx,
                               const double *__restrict__ fs, double *__restrict__ Vx_out, int batch, int N, int nx) {
  const long total = (long)batch * (N + 1) * nx;
  const int P = vxx_packed_doubles(nx);
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long kn = i / nx;
    const int r = (int)(i % nx);
    const double *f = fs + kn * nx;
    double acc = 0.0;
    if (Vxx0 && !vxx_slot_is_full((int)(kn % (N + 1)))) {
      const double *V = Vxx + kn * P;
      for (int c = 0; c < nx; ++c)
        acc += V[vxx_packed_index(nx, r, c)] * f[c];
    } else {
      const double *V = Vxx0 ? Vxx0 + kn / (N + 1) * nx * nx : Vxx + kn * nx * nx;
      for (int c = 0; c < nx; ++c) // the lower triangle mirrored (selfadjointView<Lower>, :272)
        acc += (r >= c ? V[r + (size_t)c * nx] : V[c + (size_t)r * nx]) * f[c];
    }
    Vx_out[i] = vx[i] + acc;
  }
}
// Knots [t0, t0 + nt) of instances [b0, b0 + nb) of a packed Vxx (vxx_layout.h) as full column-major blocks;
// stage knot t < N sits in factor slot (t + head) mod N, the terminal knot in slot N.
__global__ void vxx_expand_kernel(const double *__restrict__ pk, const double *__restrict__ full0, double *__restrict__ dst,
                                  int N, int nx, int head, int b0, int nb, int t0, int nt) {
  const long nn = (long)nx * nx, total = (long)nb * nt * nn;
  const int P = vxx_packed_doubles(nx);
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long kn = i / nn;
    const int e = (int)(i - kn * nn);
    const long b = b0 + kn / nt;
    const int t = t0 + (int)(kn % nt);
    const int slot = t < N ? (t + head) % N : t;
    dst[i] = vxx_slot_is_full(slot) ? full0[b * nn + e]
                                    : pk[(b * (N + 1) + slot) * P + vxx_packed_index(nx, e % nx, e / nx)];
  }
}
__global__ void fddp_quuks_kernel(const double *__restrict__ Ju, const double *__restrict__ Lu, const double *__restrict__ Vx,
                                  double *__restrict__ out, int batch, int N, int nx, int nu) {
  const long total = (long)batch * N * nu;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long kn = i / nu, b = kn / N, t = kn % N;
    const int c = (int)(i % nu);
    const double *B = Ju + kn * nx * nu + (size_t)c * nx, *v = Vx + (b * (N + 1) + t + 1) * nx;
    double acc = Lu[i];
    for (int r = 0; r < nx; ++r)
      acc += B[r] * v[r];
    out[i] = -acc;
  }
}

// one KernelEntry per compile-time shape, each defined in its own object file
// (kernel_inst.cu compiled with -DAB2_NX=.. -DAB2_NU=.. -DAB2_NC=.. -DAB2_G=..)
#define X(NX, NU, NC, G) extern const KernelEntry kEntry_##NX##_##NU##_##NC;
AB2_FOR_EACH_CONFIG(X)
#undef X
static const KernelEntry *const kTable[] = {
#define X(NX, NU, NC, G) &kEntry_##NX##_##NU##_##NC,
    AB2_FOR_EACH_CONFIG(X)
#undef X
};

static const KernelEntry *find_kernel(int nx, int nu, int nc) {
  for (const KernelEntry *e : kTable)
    if (e->nx == nx && e->nu == nu && e->nc == nc)
      return e;
  return nullptr;
}

} // namespace ab2

// ===========================================================================
// C ABI
// ===========================================================================
namespace {
thread_local std::string g_err;
int fail(int code, const std::string &msg) {
  g_err = msg;
  return code;
}
#define CUDA_TRY(expr)                                                                      \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess)                                                                  \
      return fail(AB2_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));        \
  } while (0)
// A device array the handle owns: allocated on first use (at least one element), reallocated when a larger size is
// asked for (the old contents are dropped), freed with the handle.  Reads as the pointer it holds.
template <class T> struct DevBuf {
  T *p = nullptr;
  size_t n = 0; // elements allocated
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  ~DevBuf() {
    if (p)
      cudaFree(p);
  }
  operator T *() const { return p; }
  cudaError_t ensure(size_t want) {
    if (want == 0)
      want = 1;
    if (n >= want)
      return cudaSuccess;
    if (p) {
      const cudaError_t e = cudaFree(p);
      p = nullptr;
      n = 0;
      if (e != cudaSuccess)
        return e;
    }
    const cudaError_t e = cudaMalloc(&p, want * sizeof(T));
    if (e != cudaSuccess) {
      p = nullptr;
      return e;
    }
    n = want;
    return cudaSuccess;
  }
};
} // namespace

struct ab2_gar_solver {
  ab2_gar_dims d;
  const ab2::KernelEntry *k;
  int srec, trec, nr;
  ab2::SweepParams p;
  // owned device storage
  DevBuf<double> own_stage, own_term, own_G0, own_g0;
  DevBuf<double> own_stage_sym; // triangle-packed stage records as uploaded by ab2_gar_sweep_host_sym
  DevBuf<double> gains_tmp, kkt_tmp, theta_dev, ls_tmp;
  DevBuf<double> fddp_slack, fddp_G0, fddp_g0, fddp_vx;
  DevBuf<double> inner_tmp; // [batch][2] per-instance scalars of multipliers / criterion, for host destinations
  DevBuf<double> mu_dev;    // [batch] host-given per-instance mu of the *_v sweeps, staged for the kernels
  DevBuf<double> adj_stage, adj_term, adj_g0; // the adjoint problem of ab2_gar_adjoint
  DevBuf<double> tan_rho; // rho of ab2_gar_tangent, in the solution's layouts (xs, us, vs, vsT, lam0, lams)
  DevBuf<double> ref_buf;   // ab2_gar_refine's residual (rhs layout) and correction (out layout)
  DevBuf<double> ref_norms; // staging of host norms of ab2_gar_refine / refine_many
  int nth = 0; // parameter dimension of the value function outputs (= nx in leg mode)
  int rec_nth = 0; // parameter blocks carried by the knot records (0 in leg mode)
  int legs = 0;    // >= 2: gar::ParallelRiccatiSolver (leg mode)
  bool dense = false; // gar::RiccatiSolverDense (one CTA per instance, stage-dense KKT): FF/FB have nu+nc+2nx rows
  // O(1) cycleAppend: ring heads.  fac_head: physical slot of stage knot 0 in the per-knot FACTOR arrays
  // (FF, FB, VXX, VX) -- non-zero only between a cycle_append and the next backward, which rewrites every slot
  // in place; seen by the getters only.  p.stage_head: the same for the solver-owned copy of the stage records,
  // read by the kernels through stage_slot().
  int fac_head = 0;
  DevBuf<double> cond;
  // fused pack + all-gather over peer memory (multi-GPU)
  int pg_world = 0, pg_rank = 0;
  unsigned long long pg_step = 0;
  void *pg_local = nullptr;          // cudaMalloc: [3][world][batch][per] doubles, then flags
  void *pg_peer_base[8] = {};        // IPC-opened bases (own entry = pg_local)
  ab2::PeerPtrs pg_ptrs{};
  unsigned int *pg_done = nullptr;
  size_t pg_buf_doubles = 0;
  unsigned long long pg_pushed_step = 0; // the step whose blocks the last sweep stored into the peers itself
  bool pg_in_sweep = true;               // env AB2_PEER_IN_SWEEP=0: always use the separate pack + store kernel
  DevBuf<double> out[AB2_OUT_COUNT];  // out[w].n: doubles allocated (>= out_doubles[w])
  size_t out_doubles[AB2_OUT_COUNT] = {};
  size_t out_rec[AB2_OUT_COUNT] = {};  // doubles per knot (or per instance)
  int out_knots[AB2_OUT_COUNT] = {};   // knots per instance (1 for per-instance arrays)
  DevBuf<int> status, pivstat;
  // What the handle holds.  Only the transitions below (problem_replaced, factored, rolled_out, swept_host, cycled)
  // assign these nine fields; DESIGN §1 "Handle state" tabulates them per call.
  bool have_problem = false, have_backward = false, have_forward = false;
  // ab2_gar_refine: the last backward ran on the problem's own vectors (not an adjoint / tangent problem), and the
  // trajectory outputs hold the primal solution of that factorisation (a forward since)
  bool primal_factor = false, have_primal = false;
  // ab2_gar_resolve: FB / VXX belong to the current problem (a backward ran after the last set_problem, assemble or
  // cycle_append), and the count of calls that rewrote the factorisation or the records (ab2_gar_factor_epoch)
  bool factor_current = false;
  long long epoch = 0;
  long launches = 0;
  int variant = -1;
  // Layout of out[AB2_OUT_VXX] as the last backward left it: true = packed (warp-per-instance kernel,
  // vxx_layout.h; p.Vxx0 is the full slot-0 array behind it), false = [batch][N+1][nx*nx] blocks.
  bool vxx_packed = false;
  int group_doubles[4] = {0, 0, 0, 0};
  // ab2_gar_sweep_host: internal streams, one event per stream + a fork event
  static constexpr int kPipeStreams = 4;
  cudaStream_t pipe_stream[kPipeStreams] = {};
  cudaEvent_t pipe_done[kPipeStreams] = {};
  cudaEvent_t pipe_fork = nullptr;
};

static size_t stage_total(const ab2_gar_solver *s) {
  return (size_t)s->d.batch * s->d.horizon * s->srec;
}

// The configured backward runs the warp-per-instance kernel, which stores Vxx packed.
static bool warp_kernel(const ab2_gar_solver *s) { return s->k && s->variant != 9; }

// ---- the handle's state transitions: each call that changes what the handle holds goes through these, after its
//      launches have been enqueued ----
// set_problem, assemble: new records (complete: all four arrays are held); any factorisation is stale.
static void problem_replaced(ab2_gar_solver *s, bool complete) {
  s->have_problem = complete;
  s->factor_current = false;
  s->epoch += 1;
}
// A backward rewrote every factor slot in knot order at this mu (mu_dev: a per-instance mu, which is not kept).
// primal: on the problem's own vectors, not an adjoint or tangent problem.  The trajectory outputs are stale.
static void factored(ab2_gar_solver *s, bool primal, double mueq, const double *mu_dev) {
  if (!mu_dev)
    s->p.mueq = mueq;
  s->have_backward = true;
  s->factor_current = true;
  s->primal_factor = primal;
  s->have_forward = false;
  s->have_primal = false;
  s->fac_head = 0;
  s->vxx_packed = warp_kernel(s);
  s->epoch += 1;
}
// A forward pass wrote the trajectory outputs from the last backward's factorisation.
static void rolled_out(ab2_gar_solver *s) {
  s->have_forward = true;
  s->have_primal = s->primal_factor;
}
// ab2_gar_sweep_host: new records, factored and rolled out, counted as one change of the factorisation.
static void swept_host(ab2_gar_solver *s, double mueq, const double *mu_dev) {
  s->have_problem = true;
  factored(s, true, mueq, mu_dev);
  rolled_out(s);
}
// cycle_append: the rings advanced by one knot (the parallel solver zeroed its factors instead); nothing is current.
static void cycled(ab2_gar_solver *s) {
  if (s->legs <= 1)
    s->fac_head = (s->fac_head + 1) % s->d.horizon;
  s->have_backward = false;
  s->have_forward = false;
  s->have_primal = false;
  s->factor_current = false;
  s->epoch += 1;
}

// ---- small shared pieces of the calls ----
// the copy kind of a result for the caller's memspace
static cudaMemcpyKind out_kind(int memspace) {
  return memspace == AB2_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
}
// grid of a 256-thread grid-stride kernel over n elements: at most 8 CTAs per SM
static int grid_for(const ab2_gar_solver *s, size_t n) {
  const long blocks = (long)((n + 255) / 256);
  return (int)(blocks > s->p.num_sms * 8L ? s->p.num_sms * 8L : blocks);
}
static ab2::AdjointDims adjoint_dims(const ab2_gar_solver *s) {
  const ab2_gar_dims &d = s->d;
  return ab2::AdjointDims{d.batch, d.horizon, d.nx, d.nu, d.nc, d.nct, d.nc0, s->srec, s->trec};
}
// the handle's trajectory outputs
static ab2_ls_trial trajectory(const ab2_gar_solver *s) {
  return ab2_ls_trial{s->out[AB2_OUT_XS], s->out[AB2_OUT_US],   s->out[AB2_OUT_VS],
                      s->out[AB2_OUT_VST], s->out[AB2_OUT_LBD0], s->out[AB2_OUT_LBDAS]};
}
// `count` arrays t[0 .. count) of the solution's layouts (xs .. lams, one batch each) in the handle's buffer buf
static int sol_scratch(ab2_gar_solver *s, DevBuf<double> &buf, int count, ab2_ls_trial *t) {
  const ab2_gar_dims &d = s->d;
  const size_t B = d.batch, N = d.horizon;
  const size_t n[6] = {B * (N + 1) * d.nx, B * N * d.nu, B * N * d.nc, B * d.nct, B * d.nc0, B * N * d.nx};
  const size_t one = n[0] + n[1] + n[2] + n[3] + n[4] + n[5];
  CUDA_TRY(buf.ensure(count * one));
  for (int i = 0; i < count; ++i) {
    t[i].xs = buf.p + i * one;
    t[i].us = t[i].xs + n[0];
    t[i].vs = t[i].us + n[1];
    t[i].vsT = t[i].vs + n[2];
    t[i].lam0 = t[i].vsT + n[3];
    t[i].lams = t[i].lam0 + n[4];
  }
  return AB2_OK;
}
// the SweepParams member of each output, indexed by AB2_OUT_*
static double *ab2::SweepParams::*const kOutMember[AB2_OUT_COUNT] = {
    &ab2::SweepParams::ff,   &ab2::SweepParams::fb,     &ab2::SweepParams::Vxx,     &ab2::SweepParams::vx,
    &ab2::SweepParams::ffT,  &ab2::SweepParams::fbT,    &ab2::SweepParams::kkt0,    &ab2::SweepParams::xs,
    &ab2::SweepParams::us,   &ab2::SweepParams::vs,     &ab2::SweepParams::vsT,     &ab2::SweepParams::lbd0,
    &ab2::SweepParams::lbdas, &ab2::SweepParams::fth,   &ab2::SweepParams::Vxt,     &ab2::SweepParams::Vtt,
    &ab2::SweepParams::vt,   &ab2::SweepParams::kkt0fth, &ab2::SweepParams::thGrad, &ab2::SweepParams::thHess};
// An n-double result of a call: the kernels write it at dev, which is the caller's buffer dst when that is device
// memory and the handle's scratch otherwise; copy_out() then copies the scratch to dst.
struct Staged {
  double *dst, *dev;
  size_t n;
  int copy_out(cudaStream_t st) const {
    if (dev != dst)
      CUDA_TRY(cudaMemcpyAsync(dst, dev, n * sizeof(double), cudaMemcpyDeviceToHost, st));
    return AB2_OK;
  }
};
static int stage_result(DevBuf<double> &scratch, double *dst, bool on_device, size_t n, Staged *r) {
  *r = Staged{dst, dst, n};
  if (!on_device) {
    CUDA_TRY(scratch.ensure(n));
    r->dev = scratch;
  }
  return AB2_OK;
}

extern "C" {

const char *ab2_gar_last_error(void) { return g_err.c_str(); }
const char *ab2_gar_version(void) { return "aligator_b200 gar 0.1 (sm_90a)"; }

size_t ab2_gar_stage_record_doubles(int nx, int nu, int nc) { return ab2::stage_record_len(nx, nu, nc); }
size_t ab2_gar_term_record_doubles(int nx, int nct) { return ab2::term_record_len(nx, nct); }
size_t ab2_gar_stage_record_doubles_th(int nx, int nu, int nc, int nth) {
  return ab2::stage_record_len(nx, nu, nc, nth);
}
size_t ab2_gar_term_record_doubles_th(int nx, int nct, int nth) { return ab2::term_record_len(nx, nct, nth); }
int ab2_gar_supported(int nx, int nu, int nc, int nc0) {
  if (nx < 1 || nu < 1 || nc < 0 || nc0 < 0)
    return 0;
  const ab2::KernelEntry *k = ab2::find_kernel(nx, nu, nc);
  if (k && nx + nc0 <= k->G)
    return 1; // compile-time shape, one warp (or part of one) per instance
  return ab2::block_supported(nx, nu, nc, nc0) ? 2 : 0; // run-time shape, one CTA per instance
}

static int create_impl(const ab2_gar_dims *dims, int nth, int legs, ab2_gar_solver **out);
int ab2_gar_create(const ab2_gar_dims *dims, ab2_gar_solver **out) { return create_impl(dims, 0, 0, out); }
int ab2_gar_create_parametric(const ab2_gar_dims *dims, int nth, ab2_gar_solver **out) {
  return create_impl(dims, nth, 0, out);
}
int ab2_gar_create_dense(const ab2_gar_dims *dims, ab2_gar_solver **out) { return create_impl(dims, 0, -1, out); }
int ab2_gar_create_parallel(const ab2_gar_dims *dims, int num_legs, ab2_gar_solver **out) {
  if (num_legs < 2) // parallel-solver.hxx:42-46 throws "numThreads should be greater than or equal to 2"
    return fail(AB2_ERR_INVALID, "num_legs (" + std::to_string(num_legs) + ") should be greater than or equal to 2");
  if (dims && dims->horizon + 1 < num_legs)
    return fail(AB2_ERR_INVALID, "every leg needs at least one knot: horizon + 1 >= num_legs");
  return create_impl(dims, dims ? dims->nx : 0, num_legs, out);
}

static int create_impl(const ab2_gar_dims *dims, int nth, int legs, ab2_gar_solver **out) {
  if (!dims || !out)
    return fail(AB2_ERR_INVALID, "null argument");
  const ab2_gar_dims &d = *dims;
  if (d.nx < 1 || d.nu < 1 || d.nc < 0 || d.nct < 0 || d.nc0 < 0 || d.horizon < 0 || d.batch < 1 || nth < 0)
    return fail(AB2_ERR_INVALID, "bad dimensions");
  const bool dense = legs < 0; // (legs = -1 selects the stage-dense solver)
  if (dense)
    legs = 0;
  const int rec_nth = legs > 1 ? 0 : nth; // leg mode: plain records, the parameterisation is implicit
  if (dense && !ab2::dense_supported(d.nx, d.nu, d.nc, d.nct, d.nc0))
    return fail(AB2_ERR_UNSUPPORTED, "the stage-dense KKT system (nu + nc + 2 nx rows) does not fit one CTA");
  // compile-time shapes run one warp (or part of one) per instance; every other shape runs
  // the CTA-per-instance kernel with run-time dimensions (block_kernel.cu)
  const ab2::KernelEntry *k = ab2::find_kernel(d.nx, d.nu, d.nc);
  if (k && (d.nx + d.nc0 > k->G || nth > 0))
    k = nullptr; // parametric problems run the CTA-per-instance kernel
  if (legs > 1 && !ab2::condensed_supported(d.nx, d.nc0, legs))
    return fail(AB2_ERR_UNSUPPORTED, "the condensed system of " + std::to_string(legs) + " legs does not fit one CTA's shared memory");
  if (!k && !ab2::block_supported(d.nx, d.nu, d.nc, d.nc0, nth))
    return fail(AB2_ERR_UNSUPPORTED,
                "(nx,nu,nc,nc0) = (" + std::to_string(d.nx) + "," + std::to_string(d.nu) + "," +
                    std::to_string(d.nc) + "," + std::to_string(d.nc0) +
                    ") does not fit one CTA (227 KB of shared memory, 256 rows)");
  int ndev = 0;
  CUDA_TRY(cudaGetDeviceCount(&ndev));
  if (d.device < 0 || d.device >= ndev)
    return fail(AB2_ERR_CUDA, "no such CUDA device");
  CUDA_TRY(cudaSetDevice(d.device));
  auto *s = new ab2_gar_solver();
  s->d = d;
  s->k = k;
  s->nth = nth;
  s->rec_nth = rec_nth;
  s->legs = legs;
  s->srec = (int)ab2_gar_stage_record_doubles_th(d.nx, d.nu, d.nc, rec_nth);
  if (k && k->srec_pad != s->srec) {
    delete s;
    return fail(AB2_ERR_INVALID, "internal: record size mismatch");
  }
  s->trec = (int)ab2_gar_term_record_doubles_th(d.nx, d.nct, rec_nth);
  s->nr = d.nu + d.nc + d.nx;
  s->dense = dense;
  if (dense) {
    s->k = nullptr;
    s->nr = d.nu + d.nc + 2 * d.nx; // rows of ff / fb: [k; z; l; y] (dense-kernel.hpp:28-31)
  }
  if (s->k)
    s->k->group_doubles(d.nc0, s->group_doubles);
  const int N = d.horizon, B = d.batch, nx = d.nx;
  auto setup = [&](int what, size_t rec, int knots) {
    s->out_rec[what] = rec;
    s->out_knots[what] = knots;
    s->out_doubles[what] = (size_t)B * knots * rec;
  };
  setup(AB2_OUT_FF, s->nr, N);
  setup(AB2_OUT_FB, (size_t)s->nr * nx, N);
  setup(AB2_OUT_VXX, (size_t)nx * nx, N + 1);
  setup(AB2_OUT_VX, nx, N + 1);
  setup(AB2_OUT_FFT, d.nct, 1);
  setup(AB2_OUT_FBT, (size_t)d.nct * nx, 1);
  setup(AB2_OUT_KKT0, nx + d.nc0, 1);
  setup(AB2_OUT_XS, nx, N + 1);
  setup(AB2_OUT_US, d.nu, N);
  setup(AB2_OUT_VS, d.nc, N);
  setup(AB2_OUT_VST, d.nct, 1);
  setup(AB2_OUT_LBD0, d.nc0, 1);
  setup(AB2_OUT_LBDAS, nx, N);
  setup(AB2_OUT_FTH, (size_t)s->nr * nth, N);
  setup(AB2_OUT_VXT, (size_t)nx * nth, N + 1);
  setup(AB2_OUT_VTT, (size_t)nth * nth, N + 1);
  setup(AB2_OUT_VT, nth, N + 1);
  setup(AB2_OUT_KKT0FTH, (size_t)(nx + d.nc0) * nth, 1);
  setup(AB2_OUT_THGRAD, nth, 1);
  setup(AB2_OUT_THHESS, (size_t)nth * nth, 1);
  // warp-per-instance handles: VXX holds either layout (packed + the full slot-0 array, or full blocks for variant 9)
  const size_t vxx_packed_total = (size_t)B * (N + 1) * ab2::vxx_packed_doubles(nx) + (size_t)B * nx * nx;
  // allocated and zeroed; on failure the handle is destroyed and the message names the array
  auto alloc = [&](auto &buf, size_t n, const char *what) -> int {
    cudaError_t e = buf.ensure(n);
    if (e == cudaSuccess)
      e = cudaMemset(buf.p, 0, n * sizeof(*buf.p));
    if (e != cudaSuccess) {
      ab2_gar_destroy(s);
      return fail(AB2_ERR_CUDA, std::string("cudaMalloc ") + what + ": " + cudaGetErrorString(e));
    }
    return AB2_OK;
  };
  ab2::SweepParams &p = s->p;
  std::memset(&p, 0, sizeof(p));
  for (int w = 0; w < AB2_OUT_COUNT; ++w) {
    // (+2: the forward pass of the CTA-per-instance kernel fetches odd-sized gain records
    // with 16-byte granularity, up to one double past the end of the array)
    size_t n = s->out_doubles[w];
    if (w == AB2_OUT_VXX && s->k && vxx_packed_total > n)
      n = vxx_packed_total;
    if (int rc = alloc(s->out[w], n + 2, "outputs"))
      return rc;
    p.*kOutMember[w] = s->out[w];
  }
  if (int rc = alloc(s->status, B, "status"))
    return rc;
  if (int rc = alloc(s->pivstat, B, "pivstat"))
    return rc;
  if (legs > 1)
    if (int rc = alloc(s->cond, (size_t)B * ((size_t)d.nc0 + (size_t)d.nx * (2 * legs - 1)), "cond"))
      return rc;
  p.legs = legs;
  p.cond = s->cond;
  p.N = N;
  p.nct = d.nct;
  p.nc0 = d.nc0;
  p.batch = B;
  if (s->k)
    p.Vxx0 = p.Vxx + (size_t)B * (N + 1) * ab2::vxx_packed_doubles(nx);
  p.status = s->status;
  p.pivstat = s->pivstat;
  p.nth = nth;
  p.theta = nullptr;
  {
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, d.device);
    p.num_sms = sms > 0 ? sms : 132;
  }
  if (const char *f = std::getenv("AB2_PEER_IN_SWEEP")) // 0: the exchange always runs as its own pack + store kernel
    s->pg_in_sweep = std::atoi(f) != 0;
  if (std::getenv("AB2_PHASE_CLOCKS")) { // profiling aid of the CTA-per-instance kernel: 16 phase counters
    cudaMalloc(&p.clk, 16 * sizeof(long long));
    cudaMemset(p.clk, 0, 16 * sizeof(long long));
  }
  *out = s;
  return AB2_OK;
}

int ab2_gar_destroy(ab2_gar_solver *s) {
  if (!s)
    return AB2_OK;
  cudaSetDevice(s->d.device); // (the DevBuf members are freed by delete, on this device)
  for (int w = 0; w < s->pg_world; ++w)
    if (w != s->pg_rank && s->pg_peer_base[w])
      cudaIpcCloseMemHandle(s->pg_peer_base[w]);
  if (s->pg_local)
    cudaFree(s->pg_local);
  if (s->pg_done)
    cudaFree(s->pg_done);
  for (int i = 0; i < ab2_gar_solver::kPipeStreams; ++i) {
    if (s->pipe_done[i])
      cudaEventDestroy(s->pipe_done[i]);
    if (s->pipe_stream[i])
      cudaStreamDestroy(s->pipe_stream[i]);
  }
  if (s->pipe_fork)
    cudaEventDestroy(s->pipe_fork);
  delete s;
  return AB2_OK;
}

int ab2_gar_set_tuning(ab2_gar_solver *s, const ab2_gar_tuning *t) {
  if (!s || !t)
    return fail(AB2_ERR_INVALID, "null argument");
  if (t->variant < -1 || t->variant > 10)
    return fail(AB2_ERR_INVALID, "variant must be -1 (default) or 0..10");
  if (t->variant == 9 && !ab2::block_supported(s->d.nx, s->d.nu, s->d.nc, s->d.nc0))
    return fail(AB2_ERR_UNSUPPORTED, "variant 9 (CTA per instance) does not fit this shape");
  if (t->stagger_ns < 0 || t->stagger_ns > 100000 || t->ctas_per_sm < 0 || t->ctas_per_sm > 32)
    return fail(AB2_ERR_INVALID, "stagger_ns must be in [0, 100000], ctas_per_sm in [0, 32]");
  s->variant = t->variant;
  s->p.stagger_ns = t->stagger_ns;
  s->p.ctas_per_sm = t->ctas_per_sm;
  return AB2_OK;
}

int ab2_gar_set_problem(ab2_gar_solver *s, const double *stage, const double *term, const double *G0,
                        const double *g0, int memspace, void *stream) {
  if (!s)
    return fail(AB2_ERR_INVALID, "null solver");
  CUDA_TRY(cudaSetDevice(s->d.device));
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n_stage = stage_total(s), n_term = (size_t)s->d.batch * s->trec,
               n_G0 = (size_t)s->d.batch * s->d.nc0 * s->d.nx, n_g0 = (size_t)s->d.batch * s->d.nc0;
  if (memspace == AB2_DEVICE) {
    if (stage) {
      s->p.stage = stage;
      s->p.stage_head = 0; // a caller-owned array is in knot order (the caller rotates it itself)
    }
    if (term)
      s->p.term = term;
    if (G0)
      s->p.G0 = G0;
    if (g0)
      s->p.g0 = g0;
  } else if (memspace == AB2_HOST) {
    auto up = [&](DevBuf<double> &own, const double *src, size_t n, const double *&dst) -> int {
      if (!src)
        return AB2_OK;
      CUDA_TRY(own.ensure(n));
      if (n)
        CUDA_TRY(cudaMemcpyAsync(own, src, n * sizeof(double), cudaMemcpyHostToDevice, st));
      dst = own;
      return AB2_OK;
    };
    int rc;
    if ((rc = up(s->own_stage, stage, n_stage, s->p.stage)) != AB2_OK)
      return rc;
    if (stage)
      s->p.stage_head = 0;
    if ((rc = up(s->own_term, term, n_term, s->p.term)) != AB2_OK)
      return rc;
    if ((rc = up(s->own_G0, G0, n_G0, s->p.G0)) != AB2_OK)
      return rc;
    if ((rc = up(s->own_g0, g0, n_g0, s->p.g0)) != AB2_OK)
      return rc;
  } else {
    return fail(AB2_ERR_INVALID, "memspace must be AB2_HOST or AB2_DEVICE");
  }
  problem_replaced(s, (s->p.stage && s->p.term && (s->p.G0 || s->d.nc0 == 0) && (s->p.g0 || s->d.nc0 == 0)) ||
                          (s->d.horizon == 0 && s->p.term));
  return AB2_OK;
}

// SweepParams of the instances [b0, b0 + nb) of a backward + forward launch: every array leads with the batch index.
static ab2::SweepParams slice_params(const ab2_gar_solver *s, int b0, int nb) {
  ab2::SweepParams q = s->p;
  const size_t b = (size_t)b0;
  const int N = s->d.horizon, nx = s->d.nx;
  q.batch = nb;
  q.stage += b * N * s->srec;
  q.term += b * s->trec;
  if (q.G0)
    q.G0 += b * s->d.nc0 * nx;
  if (q.g0)
    q.g0 += b * s->d.nc0;
  for (int w = 0; w < AB2_OUT_COUNT; ++w) // (the value-function outputs of nth = 0 have zero-sized records)
    if (w != AB2_OUT_VXX || !warp_kernel(s))
      q.*kOutMember[w] += b * s->out_knots[w] * s->out_rec[w];
  if (warp_kernel(s)) {
    q.Vxx += b * (N + 1) * ab2::vxx_packed_doubles(nx);
    q.Vxx0 += b * nx * nx;
  }
  q.status += b;
  q.pivstat += b;
  if (q.theta)
    q.theta += b * s->nth;
  if (q.cond)
    q.cond += b * ((size_t)s->d.nc0 + (size_t)nx * (2 * s->legs - 1));
  return q;
}

// The kernels of one (sub-)batch.  Serial solver: ONE launch (backward and/or forward).  Leg mode
// (gar::ParallelRiccatiSolver): the legs' backward recursions of all instances in one launch, the
// condensed block-tridiagonal systems in a second, the legs' rollouts in a third
// (parallel-solver.hxx:150-164, 166-203, 221-241).
static int run_kernels(ab2_gar_solver *s, ab2::SweepParams q, int bwd, int fwd, cudaStream_t st) {
  if (s->legs > 1) {
    if (bwd) {
      CUDA_TRY(cudaMemsetAsync(q.status, 0, sizeof(int) * q.batch, st)); // the legs OR / add into these
      CUDA_TRY(cudaMemsetAsync(q.pivstat, 0, sizeof(int) * q.batch, st));
      q.do_bwd = 1;
      q.do_fwd = 0;
      CUDA_TRY(ab2::launch_block(q, s->d.nx, s->d.nu, s->d.nc, st, nullptr));
      CUDA_TRY(ab2::launch_condensed(q, s->d.nx, st));
      s->launches += 2;
    }
    if (fwd) {
      q.do_bwd = 0;
      q.do_fwd = 1;
      CUDA_TRY(ab2::launch_block(q, s->d.nx, s->d.nu, s->d.nc, st, nullptr));
      s->launches += 1;
    }
    return AB2_OK;
  }
  q.do_bwd = bwd;
  q.do_fwd = fwd;
  // a forward-only launch reads Vxx in the layout the last backward wrote, whatever the tuning says now
  const bool warp = bwd ? warp_kernel(s) : s->vxx_packed;
  if (s->dense)
    CUDA_TRY(ab2::launch_dense(q, s->d.nx, s->d.nu, s->d.nc, st));
  else if (warp)
    CUDA_TRY(s->k->launch(q, s->variant == 9 ? -1 : s->variant, s->group_doubles, st, nullptr));
  else
    CUDA_TRY(ab2::launch_block(q, s->d.nx, s->d.nu, s->d.nc, st, nullptr));
  s->launches += 1;
  return AB2_OK;
}

// mueq_b: per-instance mu ([batch], device) of a *_v call, or null for the scalar mueq.  It lives in this launch's
// copy of the parameters only, so later scalar and forward-only calls never see it.
static int launch(ab2_gar_solver *s, double mueq, const double *mueq_b, int bwd, int fwd, void *stream) {
  if (!s)
    return fail(AB2_ERR_INVALID, "null solver");
  if (!s->have_problem)
    return fail(AB2_ERR_STATE, "set_problem has not been called with all four buffers");
  if (fwd && !bwd && !s->have_backward)
    return fail(AB2_ERR_STATE, "forward() before backward()");
  if (bwd && !mueq_b && !(mueq > 0.0) && (s->d.nc > 0 || s->d.nct > 0))
    return fail(AB2_ERR_INVALID, "mueq must be > 0 when constraints are present");
  CUDA_TRY(cudaSetDevice(s->d.device));
  s->p.do_bwd = bwd;
  s->p.do_fwd = fwd;
  ab2::SweepParams q = s->p;
  if (!mueq_b)
    q.mueq = mueq;
  q.mueq_b = mueq_b;
  q.peer_world = 0;
  if (bwd && s->pg_in_sweep && s->pg_peer_base[0] && s->k && s->variant != 9 && s->legs <= 1 && !s->dense &&
      s->d.horizon > 0) {
    // sharded batch: the warp-per-instance sweep stores each instance's [K0 | k0] into every rank's receive
    // buffer as soon as its backward pass is done (the exchange of step pg_step + 1)
    const unsigned long long step = s->pg_step + 1;
    const size_t total = (size_t)s->d.batch * s->d.nu * (s->d.nx + 1);
    q.peer_world = s->pg_world;
    for (int w = 0; w < s->pg_world; ++w)
      q.peer_dst[w] = s->pg_ptrs.buf[w];
    q.peer_off = (long long)((step % 3) * s->pg_world * total + (size_t)s->pg_rank * total);
    s->pg_pushed_step = step;
  }
  if (int rc = run_kernels(s, q, bwd, fwd, (cudaStream_t)stream))
    return rc;
  if (bwd)
    factored(s, true, mueq, mueq_b);
  if (fwd)
    rolled_out(s);
  return AB2_OK;
}

int ab2_gar_backward(ab2_gar_solver *s, double mueq, void *stream) { return launch(s, mueq, nullptr, 1, 0, stream); }
int ab2_gar_forward(ab2_gar_solver *s, void *stream) { return launch(s, s ? s->p.mueq : 0.0, nullptr, 0, 1, stream); }
int ab2_gar_sweep(ab2_gar_solver *s, double mueq, void *stream) { return launch(s, mueq, nullptr, 1, 1, stream); }

// A per-instance mu array of a *_v sweep as the kernels read it.  Host arrays are checked by the scalar rule (mu > 0
// when constraints are present) and staged, stream-ordered, into a buffer the handle owns; device arrays are used as
// they are (the kernels flag an unusable value with status bit ST_BAD_MU).
static int stage_mueq(ab2_gar_solver *s, const double *mueq, int memspace, cudaStream_t st, const double **dev) {
  if (!mueq)
    return fail(AB2_ERR_INVALID, "null mueq array");
  if (memspace == AB2_DEVICE) {
    *dev = mueq;
    return AB2_OK;
  }
  if (memspace != AB2_HOST)
    return fail(AB2_ERR_INVALID, "memspace must be AB2_HOST or AB2_DEVICE");
  if (s->d.nc > 0 || s->d.nct > 0)
    for (int b = 0; b < s->d.batch; ++b)
      if (!(mueq[b] > 0.0))
        return fail(AB2_ERR_INVALID, "mueq[" + std::to_string(b) + "] must be > 0 when constraints are present");
  CUDA_TRY(cudaSetDevice(s->d.device));
  CUDA_TRY(s->mu_dev.ensure(s->d.batch));
  CUDA_TRY(cudaMemcpyAsync(s->mu_dev, mueq, (size_t)s->d.batch * sizeof(double), cudaMemcpyHostToDevice, st));
  *dev = s->mu_dev;
  return AB2_OK;
}
static int launch_v(ab2_gar_solver *s, const double *mueq, int memspace, int fwd, void *stream) {
  if (!s)
    return fail(AB2_ERR_INVALID, "null solver");
  if (!s->have_problem) // (checked before anything is staged)
    return fail(AB2_ERR_STATE, "set_problem has not been called with all four buffers");
  const double *dev = nullptr;
  if (int rc = stage_mueq(s, mueq, memspace, (cudaStream_t)stream, &dev))
    return rc;
  return launch(s, 0.0, dev, 1, fwd, stream);
}
int ab2_gar_backward_v(ab2_gar_solver *s, const double *mueq, int memspace, void *stream) {
  return launch_v(s, mueq, memspace, 0, stream);
}
int ab2_gar_sweep_v(ab2_gar_solver *s, const double *mueq, int memspace, void *stream) {
  return launch_v(s, mueq, memspace, 1, stream);
}
int ab2_gar_forward_theta(ab2_gar_solver *s, const double *theta, int memspace, void *stream) {
  if (!s)
    return fail(AB2_ERR_INVALID, "null solver");
  if (theta && (s->nth == 0 || s->legs > 1))
    return fail(AB2_ERR_INVALID, "theta given to a solver without parameters (nth = 0; the parallel solver ignores theta, parallel-solver.hxx:211)");
  CUDA_TRY(cudaSetDevice(s->d.device));
  s->p.theta = nullptr;
  if (theta) {
    if (memspace == AB2_DEVICE) {
      s->p.theta = theta;
    } else {
      CUDA_TRY(s->theta_dev.ensure((size_t)s->d.batch * s->nth));
      CUDA_TRY(cudaMemcpyAsync(s->theta_dev, theta, (size_t)s->d.batch * s->nth * sizeof(double),
                               cudaMemcpyHostToDevice, (cudaStream_t)stream));
      s->p.theta = s->theta_dev;
    }
  }
  const int rc = launch(s, s->p.mueq, nullptr, 0, 1, stream);
  s->p.theta = nullptr;
  return rc;
}

// ---- argument checks and launch prologue shared by the derivative calls ----
// The fields of one argument, for the NULL and overlap checks: pointers and sizes in doubles.
struct Fields {
  const char *what;
  const char *const *names;
  const double *p[AB2_OUT_COUNT];
  size_t n[AB2_OUT_COUNT];
  int count;
};
typedef std::pair<const Fields *, const Fields *> FieldPair;
static const char *const kSolNames[6] = {"xs", "us", "vs", "vsT", "lam0", "lams"};
static const char *const kRecNames[4] = {"stage", "term", "G0", "g0"};
} // extern "C"
// the fields p, per[i] doubles per instance, `blocks` instances
static Fields make_fields(const char *what, const char *const *names, std::initializer_list<const double *> p,
                          const size_t *per, size_t blocks) {
  Fields f{what, names, {}, {}, (int)p.size()};
  int i = 0;
  for (const double *q : p) {
    f.p[i] = q;
    f.n[i] = blocks * per[i];
    ++i;
  }
  return f;
}
// the fields xs .. lams of v (an ab2_ls_iterate, ab2_ls_trial or the correction of ab2_lq_refine_work) in the
// solution's layouts, `blocks` instances (batch, or nrhs * batch)
template <class T> static Fields sol_fields(const ab2_gar_solver *s, const char *what, const T &v, size_t blocks) {
  const ab2_gar_dims &d = s->d;
  const int N = d.horizon;
  const size_t per[6] = {(size_t)(N + 1) * d.nx, (size_t)N * d.nu, (size_t)N * d.nc, (size_t)d.nct, (size_t)d.nc0,
                         (size_t)N * d.nx};
  return make_fields(what, kSolNames, {v.xs, v.us, v.vs, v.vsT, v.lam0, v.lams}, per, blocks);
}
// the fields stage, term, G0, g0 of v (an ab2_lq_grad or ab2_lq_tangent) in the problem's record layouts
template <class T> static Fields rec_fields(const ab2_gar_solver *s, const char *what, const T &v, size_t blocks) {
  const ab2_gar_dims &d = s->d;
  const size_t per[4] = {(size_t)d.horizon * s->srec, (size_t)s->trec, (size_t)d.nc0 * d.nx, (size_t)d.nc0};
  return make_fields(what, kRecNames, {v.stage, v.term, v.G0, v.g0}, per, blocks);
}
static int require(const Fields &f, const char *who) {
  for (int i = 0; i < f.count; ++i)
    if (f.n[i] && !f.p[i])
      return fail(AB2_ERR_INVALID, std::string(who) + ": " + f.what + " " + f.names[i] + " is NULL");
  return AB2_OK;
}
// no field of a may overlap a field of b (a and b the same argument: two different fields of it)
static int refuse_overlap(const Fields &a, const Fields &b, const char *who) {
  for (int i = 0; i < a.count; ++i)
    for (int o = &a == &b ? i + 1 : 0; o < b.count; ++o)
      if (a.p[i] && b.p[o] && a.n[i] && b.n[o] && a.p[i] < b.p[o] + b.n[o] && b.p[o] < a.p[i] + a.n[i])
        return fail(AB2_ERR_INVALID, std::string(who) + ": " + a.what + " " + a.names[i] + " overlaps " + b.what + " " +
                                         b.names[o]);
  return AB2_OK;
}
static const char *const kRhsNames[6] = {"q", "r", "d", "dN", "g0", "f"};
// the fields q .. f of v (an ab2_lq_rhs or the residual of ab2_lq_refine_work) in resolve's rhs layouts (the same
// sizes as the solution's)
template <class T> static Fields rhs_fields(const ab2_gar_solver *s, const char *what, const T &v, size_t blocks) {
  Fields f = sol_fields(s, what, ab2_ls_iterate{v.q, v.r, v.d, v.dN, v.g0, v.f}, blocks);
  f.names = kRhsNames;
  return f;
}
static const char *const kFacNames[6] = {"ff", "fb", "vxx", "vx", "fft", "fbt"};
// the fields of v (an ab2_factor_cotangent or ab2_factor_tangent) in ab2_gar_get's layouts of the factorisation
// (FF .. FBT, vxx as full blocks)
template <class T> static Fields fac_fields(const ab2_gar_solver *s, const char *what, const T &v, size_t blocks) {
  const ab2_gar_dims &d = s->d;
  const size_t N = d.horizon, nx = d.nx, nr = d.nu + d.nc + d.nx;
  const size_t per[6] = {N * nr, N * nr * nx, (N + 1) * nx * nx, (N + 1) * nx, (size_t)d.nct, (size_t)d.nct * nx};
  return make_fields(what, kFacNames, {v.ff, v.fb, v.vxx, v.vx, v.fft, v.fbt}, per, blocks);
}
extern "C" {
static const char *const kOutNames[AB2_OUT_COUNT] = {"FF",   "FB",    "VXX",  "VX",  "FFT",     "FBT",    "KKT0",
                                                     "XS",   "US",    "VS",   "VST", "LBD0",    "LBDAS",  "FTH",
                                                     "VXT",  "VTT",   "VT",   "KKT0FTH", "THGRAD", "THHESS"};
// the handle's own output arrays, as allocated
static Fields out_fields(const ab2_gar_solver *s) {
  Fields f{"the handle's output", kOutNames, {}, {}, AB2_OUT_COUNT};
  for (int w = 0; w < AB2_OUT_COUNT; ++w) {
    f.p[w] = s->out[w];
    f.n[w] = s->out[w].n;
  }
  return f;
}
// the scalar mu rule (a per-instance array is checked when it is staged)
static int check_mu(const ab2_gar_solver *s, double mueq, const double *mueq_arr, const char *who) {
  if (!mueq_arr && !(mueq > 0.0) && (s->d.nc > 0 || s->d.nct > 0))
    return fail(AB2_ERR_INVALID, std::string(who) + ": mueq must be > 0 when constraints are present");
  return AB2_OK;
}
// The prologue of a call whose arguments have been checked: the handle's device, the caller's stream (*st) and the
// per-instance mu mueq_arr (in memspace) as the kernels read it (*mu_dev; null for the scalar mu).
static int begin_launch(ab2_gar_solver *s, const double *mueq_arr, int memspace, void *stream, cudaStream_t *st,
                        const double **mu_dev) {
  CUDA_TRY(cudaSetDevice(s->d.device));
  *st = (cudaStream_t)stream;
  *mu_dev = nullptr;
  return mueq_arr ? stage_mueq(s, mueq_arr, memspace, *st, mu_dev) : AB2_OK;
}

// ---- adjoint of the LQ solve: records kernel (lq_adjoint.cu), the sweep on the adjoint problem, gradient kernel
//      (lq_jacobian.cu) ----
// The handle checks shared by ab2_gar_adjoint and ab2_gar_tangent, in this order: handle kind, problem set.
static int check_solve_handle(const ab2_gar_solver *s, const char *who) {
  if (s->nth > 0 || s->legs > 1)
    return fail(AB2_ERR_UNSUPPORTED, std::string(who) + ": parametric (nth > 0) and parallel handles are not supported");
  if (!s->have_problem)
    return fail(AB2_ERR_STATE, std::string(who) + ": set_problem has not been called with all four buffers");
  return AB2_OK;
}

// The current problem's matrices with the vectors q, r, d, f, q_N, d_N, g0 = -cot (copy: = cot), solved by the
// handle's own sweep (two launches).  mu_dev: the staged per-instance mu, or null for the scalar mueq.
static int solve_cotangent_problem(ab2_gar_solver *s, double mueq, const double *mu_dev, const ab2_ls_iterate *cot,
                                   bool copy, cudaStream_t st) {
  const size_t B = s->d.batch;
  CUDA_TRY(s->adj_stage.ensure(stage_total(s)));
  CUDA_TRY(s->adj_term.ensure(B * s->trec));
  CUDA_TRY(s->adj_g0.ensure(B * s->d.nc0));
  // 1. the problem: same matrices, vectors = -cot (copy: cot)
  ab2::AdjointRecordArgs ra{adjoint_dims(s), s->p.stage_head, s->p.stage, s->p.term, cot->xs, cot->us, cot->vs,
                            cot->vsT, cot->lam0, cot->lams, s->adj_stage, s->adj_term, s->adj_g0, copy};
  CUDA_TRY(ab2::launch_adjoint_records(ra, st));
  s->launches += 1;
  // 2. backward + forward on it; the problem pointers change in this launch's copy of the parameters only, and a
  //    sharded handle never publishes these gains to its peers
  ab2::SweepParams q = s->p;
  if (!mu_dev)
    q.mueq = mueq;
  q.stage = s->adj_stage;
  q.stage_head = 0;
  q.term = s->adj_term;
  q.g0 = s->adj_g0;
  q.mueq_b = mu_dev;
  q.peer_world = 0;
  if (int rc = run_kernels(s, q, 1, 1, st))
    return rc;
  factored(s, false, mueq, mu_dev); // the trajectory outputs are w or zdot, not the primal solution
  rolled_out(s);
  return AB2_OK;
}

// mueq_arr: the per-instance mu of ab2_gar_adjoint_v (memspace), or null for the scalar mueq.
static int adjoint_impl(ab2_gar_solver *s, double mueq, const double *mueq_arr, int memspace,
                        const ab2_ls_iterate *primal, const ab2_ls_iterate *cot, const ab2_lq_grad *grad, void *stream) {
  if (!s || !primal || !cot || !grad)
    return fail(AB2_ERR_INVALID, "null argument");
  const char *who = "adjoint";
  if (int rc = check_solve_handle(s, who))
    return rc;
  // the gradient kernel reads the primal after the sweep has overwritten the handle's outputs
  const Fields P = sol_fields(s, "primal", *primal, s->d.batch);
  if (int rc = require(P, who))
    return rc;
  if (int rc = refuse_overlap(P, out_fields(s), who))
    return rc;
  if (int rc = check_mu(s, mueq, mueq_arr, who))
    return rc;
  cudaStream_t st;
  const double *mu_dev;
  if (int rc = begin_launch(s, mueq_arr, memspace, stream, &st, &mu_dev))
    return rc;
  // 1. + 2. the adjoint problem (vectors = -cotangent) and its solve
  if (int rc = solve_cotangent_problem(s, mueq, mu_dev, cot, false, st))
    return rc;
  // 3. gradient records from the primal z and the adjoint w (the trajectory outputs): dh = -w, dK = -w z^T
  const ab2_ls_trial w = trajectory(s);
  ab2::JacobianGradArgs ga{adjoint_dims(s), 1,
                           primal->xs, primal->us, primal->vs, primal->vsT, primal->lam0, primal->lams,
                           w.xs, w.us, w.vs, w.vsT, w.lam0, w.lams,
                           grad->stage, grad->term, grad->G0, grad->g0, true};
  CUDA_TRY(ab2::launch_jacobian_grad(ga, st));
  s->launches += 1;
  return AB2_OK;
}
int ab2_gar_adjoint(ab2_gar_solver *s, double mueq, const ab2_ls_iterate *primal, const ab2_ls_iterate *cotangent,
                    const ab2_lq_grad *grad, void *stream) {
  return adjoint_impl(s, mueq, nullptr, AB2_DEVICE, primal, cotangent, grad, stream);
}
int ab2_gar_adjoint_v(ab2_gar_solver *s, const double *mueq, int memspace, const ab2_ls_iterate *primal,
                      const ab2_ls_iterate *cotangent, const ab2_lq_grad *grad, void *stream) {
  if (!mueq)
    return fail(AB2_ERR_INVALID, "null mueq array");
  return adjoint_impl(s, 0.0, mueq, memspace, primal, cotangent, grad, stream);
}

// ---- tangent of the LQ solve: right-hand-side kernel (lq_jacobian.cu), then the adjoint's records kernel and sweep ----
static int tangent_impl(ab2_gar_solver *s, double mueq, const double *mueq_arr, int memspace,
                        const ab2_ls_iterate *primal, const ab2_lq_tangent *dot, void *stream) {
  if (!s || !primal || !dot)
    return fail(AB2_ERR_INVALID, "null argument");
  const char *who = "tangent";
  if (int rc = check_solve_handle(s, who))
    return rc;
  // the primal is read completely by the first launch, before the sweep writes any output: it may alias them
  if (int rc = require(sol_fields(s, "primal", *primal, s->d.batch), who))
    return rc;
  if (int rc = check_mu(s, mueq, mueq_arr, who))
    return rc;
  cudaStream_t st;
  const double *mu_dev;
  if (int rc = begin_launch(s, mueq_arr, memspace, stream, &st, &mu_dev))
    return rc;
  ab2_ls_trial rho;
  if (int rc = sol_scratch(s, s->tan_rho, 1, &rho))
    return rc;
  // 1. rho = Kdot z + hdot, in the solution's layouts
  ab2::JacobianRhsArgs ra{adjoint_dims(s), 1, dot->stage, dot->term, dot->G0, dot->g0,
                          primal->xs, primal->us, primal->vs, primal->vsT, primal->lam0, primal->lams,
                          rho.xs, rho.us, rho.vs, rho.vsT, rho.lam0, rho.lams};
  CUDA_TRY(ab2::launch_jacobian_rhs(ra, st));
  s->launches += 1;
  // 2. + 3. the tangent problem (vectors = rho) and its solve: the trajectory outputs become zdot
  const ab2_ls_iterate rho_in{rho.xs, rho.us, rho.vs, rho.vsT, rho.lam0, rho.lams};
  return solve_cotangent_problem(s, mueq, mu_dev, &rho_in, true, st);
}
int ab2_gar_tangent(ab2_gar_solver *s, double mueq, const ab2_ls_iterate *primal, const ab2_lq_tangent *dot,
                    void *stream) {
  return tangent_impl(s, mueq, nullptr, AB2_DEVICE, primal, dot, stream);
}
int ab2_gar_tangent_v(ab2_gar_solver *s, const double *mueq, int memspace, const ab2_ls_iterate *primal,
                      const ab2_lq_tangent *dot, void *stream) {
  if (!mueq)
    return fail(AB2_ERR_INVALID, "null mueq array");
  return tangent_impl(s, 0.0, mueq, memspace, primal, dot, stream);
}

// ---- re-solve for new vectors (lq_resolve.cu): the vector half of the recursion on the last backward's factorisation ----
// The first checks of every call that runs resolve's program, in this order: handle kind, factorisation current, nrhs.
static int check_resolve_handle(const ab2_gar_solver *s, int nrhs, const char *who) {
  if (s->nth > 0 || s->legs > 1 || s->dense)
    return fail(AB2_ERR_UNSUPPORTED, std::string(who) + ": dense, parametric (nth > 0) and parallel handles are not supported");
  if (!s->have_problem || !s->factor_current)
    return fail(AB2_ERR_STATE, std::string(who) + ": no backward since the last set_problem, assemble or cycle_append");
  if (nrhs < 0)
    return fail(AB2_ERR_INVALID, std::string(who) + ": nrhs < 0");
  return AB2_OK;
}
static int check_resolve_fits(const ab2_gar_solver *s, const char *who) {
  const ab2_gar_dims &d = s->d;
  if ((size_t)ab2::resolve_item_doubles(d.nx, d.nu, d.nc, d.nc0, 1) * sizeof(double) > ab2::kResolveSmemMax)
    return fail(AB2_ERR_UNSUPPORTED, std::string(who) + ": one right-hand side of this shape does not fit 227 KB of shared memory");
  return AB2_OK;
}
// The records and the last backward's factorisation as resolve's program reads them (no right-hand sides).
static ab2::ResolveArgs factor_view(const ab2_gar_solver *s, double mueq, const double *mu_dev) {
  const ab2_gar_dims &d = s->d;
  ab2::ResolveArgs a{};
  a.batch = d.batch;
  a.N = d.horizon;
  a.nx = d.nx;
  a.nu = d.nu;
  a.nc = d.nc;
  a.nct = d.nct;
  a.nc0 = d.nc0;
  a.srec = s->srec;
  a.trec = s->trec;
  a.stage_head = s->p.stage_head;
  a.stage = s->p.stage;
  a.term = s->p.term;
  a.G0 = s->p.G0;
  a.fb = s->out[AB2_OUT_FB];
  a.fbT = s->out[AB2_OUT_FBT];
  a.Vxx = s->out[AB2_OUT_VXX];
  a.Vxx0 = s->vxx_packed ? s->p.Vxx0 : nullptr;
  a.mueq = mueq;
  a.mueq_b = mu_dev;
  return a;
}
// resolve's program on the handle's current factorisation, rhs -> out (one launch).  mu_dev: the staged per-instance
// mu, or null for the scalar mueq.
static int run_resolve(ab2_gar_solver *s, double mueq, const double *mu_dev, int nrhs, const ab2_lq_rhs *rhs,
                       const ab2_ls_trial *out, cudaStream_t st) {
  ab2::ResolveArgs a = factor_view(s, mueq, mu_dev);
  a.nrhs = nrhs;
  a.q = rhs->q;
  a.r = rhs->r;
  a.d = rhs->d;
  a.dN = rhs->dN;
  a.g0 = rhs->g0;
  a.f = rhs->f;
  a.xs = out->xs;
  a.us = out->us;
  a.vs = out->vs;
  a.vsT = out->vsT;
  a.lam0 = out->lam0;
  a.lams = out->lams;
  CUDA_TRY(ab2::launch_resolve(a, st));
  s->launches += 1;
  return AB2_OK;
}
static int resolve_impl(ab2_gar_solver *s, double mueq, const double *mueq_arr, int memspace, int nrhs,
                        const ab2_lq_rhs *rhs, const ab2_ls_trial *out, void *stream) {
  if (!s || !rhs || !out)
    return fail(AB2_ERR_INVALID, "null argument");
  const char *who = "resolve";
  if (int rc = check_resolve_handle(s, nrhs, who))
    return rc;
  const size_t R = (size_t)nrhs * s->d.batch;
  if (int rc = require(sol_fields(s, "out", *out, 1), who)) // (refused even at nrhs = 0)
    return rc;
  if (int rc = check_mu(s, mueq, mueq_arr, who))
    return rc;
  // the backward pass parks its per-knot vectors in the out arrays before it has read every rhs entry: an out array
  // that overlaps an rhs array would be read after it was overwritten
  if (int rc = refuse_overlap(rhs_fields(s, "rhs", *rhs, R), sol_fields(s, "out", *out, R), who))
    return rc;
  if (int rc = check_resolve_fits(s, who))
    return rc;
  if (nrhs == 0)
    return AB2_OK;
  cudaStream_t st;
  const double *mu_dev;
  if (int rc = begin_launch(s, mueq_arr, memspace, stream, &st, &mu_dev))
    return rc;
  return run_resolve(s, mueq, mu_dev, nrhs, rhs, out, st);
}
int ab2_gar_resolve(ab2_gar_solver *s, double mueq, int nrhs, const ab2_lq_rhs *rhs, const ab2_ls_trial *out,
                    void *stream) {
  return resolve_impl(s, mueq, nullptr, AB2_DEVICE, nrhs, rhs, out, stream);
}
int ab2_gar_resolve_v(ab2_gar_solver *s, const double *mueq, int memspace, int nrhs, const ab2_lq_rhs *rhs,
                      const ab2_ls_trial *out, void *stream) {
  if (!mueq)
    return fail(AB2_ERR_INVALID, "null mueq array");
  return resolve_impl(s, 0.0, mueq, memspace, nrhs, rhs, out, stream);
}

// ---- derivatives of a parametric solution with respect to theta (lq_theta.cu): J d and J^T zbar from the stored
//      factors, one launch each ----
static const char *const kThetaNames[1] = {"theta"};
// a [blocks][nth] theta array as one field
static Fields theta_fields(const ab2_gar_solver *s, const char *what, const double *p, size_t blocks) {
  const size_t per[1] = {(size_t)s->nth};
  return make_fields(what, kThetaNames, {p}, per, blocks);
}
// The checks both calls share, in this order: handle kind, factorisation current, nrhs, then that one direction fits.
static int check_theta_handle(const ab2_gar_solver *s, int nrhs, const char *who) {
  if (s->nth == 0 || s->legs > 1 || s->dense)
    return fail(AB2_ERR_UNSUPPORTED, std::string(who) + ": handles without parameters (nth = 0, dense) and parallel handles are not supported");
  if (!s->have_problem || !s->factor_current)
    return fail(AB2_ERR_STATE, std::string(who) + ": no backward since the last set_problem or assemble");
  if (nrhs < 0)
    return fail(AB2_ERR_INVALID, std::string(who) + ": nrhs < 0");
  return AB2_OK;
}
static int check_theta_fits(const ab2_gar_solver *s, const char *who) {
  const ab2_gar_dims &d = s->d;
  if ((size_t)ab2::theta_item_doubles(d.nx, d.nu, d.nc, d.nct, d.nc0, s->nth, 1) * sizeof(double) > ab2::kThetaSmemMax)
    return fail(AB2_ERR_UNSUPPORTED, std::string(who) + ": one direction of this shape does not fit 227 KB of shared memory");
  return AB2_OK;
}
// The stored factorisation as the theta programs read it (parametric handles run the CTA kernel: full VXX blocks).
static ab2::ThetaArgs theta_view(const ab2_gar_solver *s, int nrhs) {
  const ab2_gar_dims &d = s->d;
  ab2::ThetaArgs a{};
  a.batch = d.batch;
  a.N = d.horizon;
  a.nx = d.nx;
  a.nu = d.nu;
  a.nc = d.nc;
  a.nct = d.nct;
  a.nc0 = d.nc0;
  a.nth = s->nth;
  a.nrhs = nrhs;
  a.fb = s->out[AB2_OUT_FB];
  a.fth = s->out[AB2_OUT_FTH];
  a.fbT = s->out[AB2_OUT_FBT];
  a.Vxx = s->out[AB2_OUT_VXX];
  a.Vxt = s->out[AB2_OUT_VXT];
  a.kkt0fth = s->out[AB2_OUT_KKT0FTH];
  return a;
}
int ab2_gar_theta_tangent(ab2_gar_solver *s, int nrhs, const double *dtheta, const ab2_ls_trial *out, void *stream) {
  if (!s || !out)
    return fail(AB2_ERR_INVALID, "null argument");
  const char *who = "theta_tangent";
  if (int rc = check_theta_handle(s, nrhs, who))
    return rc;
  const size_t R = (size_t)nrhs * s->d.batch;
  const Fields O = sol_fields(s, "out", *out, R), T = theta_fields(s, "dtheta", dtheta, R);
  if (int rc = require(sol_fields(s, "out", *out, 1), who)) // (refused even at nrhs = 0)
    return rc;
  if (int rc = require(theta_fields(s, "dtheta", dtheta, 1), who))
    return rc;
  if (int rc = refuse_overlap(T, O, who))
    return rc;
  if (int rc = refuse_overlap(O, out_fields(s), who))
    return rc;
  if (int rc = check_theta_fits(s, who))
    return rc;
  if (nrhs == 0)
    return AB2_OK;
  CUDA_TRY(cudaSetDevice(s->d.device));
  ab2::ThetaArgs a = theta_view(s, nrhs);
  a.dtheta = dtheta;
  a.xs = out->xs;
  a.us = out->us;
  a.vs = out->vs;
  a.vsT = out->vsT;
  a.lam0 = out->lam0;
  a.lams = out->lams;
  CUDA_TRY(ab2::launch_theta_tangent(a, (cudaStream_t)stream));
  s->launches += 1;
  return AB2_OK;
}
int ab2_gar_theta_adjoint(ab2_gar_solver *s, int nrhs, const ab2_ls_iterate *cot, double *theta_bar, void *stream) {
  if (!s || !cot)
    return fail(AB2_ERR_INVALID, "null argument");
  const char *who = "theta_adjoint";
  if (int rc = check_theta_handle(s, nrhs, who))
    return rc;
  const size_t R = (size_t)nrhs * s->d.batch;
  const Fields T = theta_fields(s, "theta_bar", theta_bar, R);
  if (int rc = require(theta_fields(s, "theta_bar", theta_bar, 1), who)) // (refused even at nrhs = 0)
    return rc;
  if (int rc = refuse_overlap(sol_fields(s, "cot", *cot, R), T, who))
    return rc;
  if (int rc = refuse_overlap(T, out_fields(s), who))
    return rc;
  if (int rc = check_theta_fits(s, who))
    return rc;
  if (nrhs == 0)
    return AB2_OK;
  CUDA_TRY(cudaSetDevice(s->d.device));
  ab2::ThetaArgs a = theta_view(s, nrhs);
  a.cxs = cot->xs;
  a.cus = cot->us;
  a.cvs = cot->vs;
  a.cvsT = cot->vsT;
  a.clam0 = cot->lam0;
  a.clams = cot->lams;
  a.theta_bar = theta_bar;
  CUDA_TRY(ab2::launch_theta_adjoint(a, (cudaStream_t)stream));
  s->launches += 1;
  return AB2_OK;
}
// ---- derivatives of the backward recursion (lq_factor_adjoint.cu, lq_factor_tangent.cu) ----
// The handle checks ab2_gar_factor_adjoint and ab2_gar_factor_tangent share: handle kind, and a backward on the
// problem's own vectors.
static int check_factor_handle(const ab2_gar_solver *s, const char *who) {
  if (int rc = check_resolve_handle(s, 0, who))
    return rc;
  if (!s->primal_factor)
    return fail(AB2_ERR_STATE, std::string(who) + ": FF and VX hold an adjoint or tangent solve; run a backward first");
  return AB2_OK;
}

// ---- reverse mode of the backward recursion (lq_factor_adjoint.cu): cotangents of the factorisation -> gradients ----
static int factor_adjoint_impl(ab2_gar_solver *s, double mueq, const double *mueq_arr, int memspace,
                               const ab2_factor_cotangent *cot, const ab2_lq_grad *grad, void *stream) {
  if (!s || !cot || !grad)
    return fail(AB2_ERR_INVALID, "null argument");
  const char *who = "factor_adjoint";
  if (int rc = check_factor_handle(s, who))
    return rc;
  if (int rc = check_mu(s, mueq, mueq_arr, who))
    return rc;
  // the gradients are written knot by knot while later knots' cotangents and factors are still to be read
  const ab2_gar_dims &d = s->d;
  const Fields G = rec_fields(s, "grad", *grad, d.batch);
  if (int rc = refuse_overlap(G, fac_fields(s, "cotangent", *cot, d.batch), who))
    return rc;
  if (int rc = refuse_overlap(G, out_fields(s), who))
    return rc;
  if ((size_t)ab2::factor_adjoint_item_doubles(d.nx, d.nu, d.nc) * sizeof(double) > ab2::kFactorAdjointSmemMax)
    return fail(AB2_ERR_UNSUPPORTED, std::string(who) + ": one instance of this shape does not fit 227 KB of shared memory");
  cudaStream_t st;
  const double *mu_dev;
  if (int rc = begin_launch(s, mueq_arr, memspace, stream, &st, &mu_dev))
    return rc;
  ab2::FactorAdjointArgs a{};
  a.fac = factor_view(s, mueq, mu_dev);
  a.ff = s->out[AB2_OUT_FF];
  a.vx = s->out[AB2_OUT_VX];
  a.ffT = s->out[AB2_OUT_FFT];
  a.c_ff = cot->ff;
  a.c_fb = cot->fb;
  a.c_vxx = cot->vxx;
  a.c_vx = cot->vx;
  a.c_fft = cot->fft;
  a.c_fbt = cot->fbt;
  a.g_stage = grad->stage;
  a.g_term = grad->term;
  a.g_G0 = grad->G0;
  a.g_g0 = grad->g0;
  CUDA_TRY(ab2::launch_factor_adjoint(a, st));
  s->launches += 1;
  return AB2_OK;
}
int ab2_gar_factor_adjoint(ab2_gar_solver *s, double mueq, const ab2_factor_cotangent *cot, const ab2_lq_grad *grad,
                           void *stream) {
  return factor_adjoint_impl(s, mueq, nullptr, AB2_DEVICE, cot, grad, stream);
}
int ab2_gar_factor_adjoint_v(ab2_gar_solver *s, const double *mueq, int memspace, const ab2_factor_cotangent *cot,
                             const ab2_lq_grad *grad, void *stream) {
  if (!mueq)
    return fail(AB2_ERR_INVALID, "null mueq array");
  return factor_adjoint_impl(s, 0.0, mueq, memspace, cot, grad, stream);
}

// ---- forward mode of the backward recursion (lq_factor_tangent.cu): tangent records -> tangents of the factorisation ----
static int factor_tangent_impl(ab2_gar_solver *s, double mueq, const double *mueq_arr, int memspace,
                               const ab2_lq_tangent *dot, const ab2_factor_tangent *out, void *stream) {
  if (!s || !dot || !out)
    return fail(AB2_ERR_INVALID, "null argument");
  const char *who = "factor_tangent";
  if (int rc = check_factor_handle(s, who))
    return rc;
  if (int rc = check_mu(s, mueq, mueq_arr, who))
    return rc;
  // the tangents are written knot by knot while later knots' tangent records and factors are still to be read
  const ab2_gar_dims &d = s->d;
  const Fields O = fac_fields(s, "out", *out, d.batch);
  if (int rc = refuse_overlap(O, rec_fields(s, "tangent", *dot, d.batch), who))
    return rc;
  if (int rc = refuse_overlap(O, out_fields(s), who))
    return rc;
  if ((size_t)ab2::factor_tangent_item_doubles(d.nx, d.nu, d.nc) * sizeof(double) > ab2::kFactorTangentSmemMax)
    return fail(AB2_ERR_UNSUPPORTED, std::string(who) + ": one instance of this shape does not fit 227 KB of shared memory");
  cudaStream_t st;
  const double *mu_dev;
  if (int rc = begin_launch(s, mueq_arr, memspace, stream, &st, &mu_dev))
    return rc;
  ab2::FactorTangentArgs a{};
  a.fac = factor_view(s, mueq, mu_dev);
  a.ff = s->out[AB2_OUT_FF];
  a.vx = s->out[AB2_OUT_VX];
  a.ffT = s->out[AB2_OUT_FFT];
  a.d_stage = dot->stage;
  a.d_term = dot->term;
  a.o_ff = out->ff;
  a.o_fb = out->fb;
  a.o_vxx = out->vxx;
  a.o_vx = out->vx;
  a.o_fft = out->fft;
  a.o_fbt = out->fbt;
  CUDA_TRY(ab2::launch_factor_tangent(a, st));
  s->launches += 1;
  return AB2_OK;
}
int ab2_gar_factor_tangent(ab2_gar_solver *s, double mueq, const ab2_lq_tangent *dot, const ab2_factor_tangent *out,
                           void *stream) {
  return factor_tangent_impl(s, mueq, nullptr, AB2_DEVICE, dot, out, stream);
}
int ab2_gar_factor_tangent_v(ab2_gar_solver *s, const double *mueq, int memspace, const ab2_lq_tangent *dot,
                             const ab2_factor_tangent *out, void *stream) {
  if (!mueq)
    return fail(AB2_ERR_INVALID, "null mueq array");
  return factor_tangent_impl(s, 0.0, mueq, memspace, dot, out, stream);
}

int ab2_gar_factor_epoch(const ab2_gar_solver *s, long long *epoch) {
  if (!s || !epoch)
    return fail(AB2_ERR_INVALID, "null argument");
  *epoch = s->epoch;
  return AB2_OK;
}

// ---- Jacobians (lq_jacobian.cu): many cotangents or tangents on the last backward's factorisation, through resolve ----

static int adjoint_many_impl(ab2_gar_solver *s, double mueq, const double *mueq_arr, int memspace, int nrhs,
                             const ab2_ls_iterate *primal, const ab2_ls_iterate *cot, const ab2_ls_trial *work,
                             const ab2_lq_grad *grad, void *stream) {
  const char *who = "adjoint_many";
  if (!s || !primal || !cot || !work || !grad)
    return fail(AB2_ERR_INVALID, "null argument");
  if (int rc = check_resolve_handle(s, nrhs, who))
    return rc;
  const ab2_gar_dims &d = s->d;
  const size_t B = d.batch, R = (size_t)nrhs * B;
  const Fields P = sol_fields(s, "primal", *primal, B), Z = sol_fields(s, "cotangent", *cot, R),
               W = sol_fields(s, "work", *work, R), G = rec_fields(s, "grad", *grad, R);
  if (int rc = require(W, who))
    return rc;
  if (int rc = require(P, who))
    return rc;
  if (int rc = check_mu(s, mueq, mueq_arr, who))
    return rc;
  // resolve writes work while it reads the cotangent; the gradient kernel then reads work and the primal
  for (const FieldPair &ab : {FieldPair{&Z, &W}, FieldPair{&W, &P}, FieldPair{&G, &P}, FieldPair{&G, &W},
                              FieldPair{&G, &G}})
    if (int rc = refuse_overlap(*ab.first, *ab.second, who))
      return rc;
  if (int rc = check_resolve_fits(s, who))
    return rc;
  if (nrhs == 0)
    return AB2_OK;
  cudaStream_t st;
  const double *mu_dev;
  if (int rc = begin_launch(s, mueq_arr, memspace, stream, &st, &mu_dev))
    return rc;
  // 1. y_j = resolve(zbar_j) = -K^-1 zbar_j: the cotangent fields are resolve's rhs fields
  const ab2_lq_rhs rhs{cot->xs, cot->us, cot->vs, cot->vsT, cot->lam0, cot->lams};
  if (int rc = run_resolve(s, mueq, mu_dev, nrhs, &rhs, work, st))
    return rc;
  // 2. gradient records from y_j and z
  ab2::JacobianGradArgs ga{adjoint_dims(s), nrhs,
                           primal->xs, primal->us, primal->vs, primal->vsT, primal->lam0, primal->lams,
                           work->xs, work->us, work->vs, work->vsT, work->lam0, work->lams,
                           grad->stage, grad->term, grad->G0, grad->g0, false};
  CUDA_TRY(ab2::launch_jacobian_grad(ga, st));
  s->launches += 1;
  return AB2_OK;
}
int ab2_gar_adjoint_many(ab2_gar_solver *s, double mueq, int nrhs, const ab2_ls_iterate *primal,
                         const ab2_ls_iterate *cotangent, const ab2_ls_trial *work, const ab2_lq_grad *grad,
                         void *stream) {
  return adjoint_many_impl(s, mueq, nullptr, AB2_DEVICE, nrhs, primal, cotangent, work, grad, stream);
}
int ab2_gar_adjoint_many_v(ab2_gar_solver *s, const double *mueq, int memspace, int nrhs, const ab2_ls_iterate *primal,
                           const ab2_ls_iterate *cotangent, const ab2_ls_trial *work, const ab2_lq_grad *grad,
                           void *stream) {
  if (!mueq)
    return fail(AB2_ERR_INVALID, "null mueq array");
  return adjoint_many_impl(s, 0.0, mueq, memspace, nrhs, primal, cotangent, work, grad, stream);
}

static int tangent_many_impl(ab2_gar_solver *s, double mueq, const double *mueq_arr, int memspace, int nrhs,
                             const ab2_ls_iterate *primal, const ab2_lq_tangent *dot, const ab2_ls_trial *work,
                             const ab2_ls_trial *out, void *stream) {
  const char *who = "tangent_many";
  if (!s || !primal || !dot || !work || !out)
    return fail(AB2_ERR_INVALID, "null argument");
  if (int rc = check_resolve_handle(s, nrhs, who))
    return rc;
  const ab2_gar_dims &d = s->d;
  const size_t B = d.batch, R = (size_t)nrhs * B;
  const Fields P = sol_fields(s, "primal", *primal, B), D = rec_fields(s, "dot", *dot, R),
               W = sol_fields(s, "work", *work, R), O = sol_fields(s, "out", *out, R);
  if (int rc = require(W, who))
    return rc;
  if (int rc = require(O, who))
    return rc;
  if (int rc = require(P, who))
    return rc;
  if (int rc = check_mu(s, mueq, mueq_arr, who))
    return rc;
  // the rho kernel writes work while it reads the tangent and the primal; resolve then writes out while it reads work
  for (const FieldPair &ab : {FieldPair{&D, &W}, FieldPair{&P, &W}, FieldPair{&W, &O}, FieldPair{&O, &P},
                              FieldPair{&O, &O}})
    if (int rc = refuse_overlap(*ab.first, *ab.second, who))
      return rc;
  if (int rc = check_resolve_fits(s, who))
    return rc;
  if (nrhs == 0)
    return AB2_OK;
  cudaStream_t st;
  const double *mu_dev;
  if (int rc = begin_launch(s, mueq_arr, memspace, stream, &st, &mu_dev))
    return rc;
  // 1. rho_j = Kdot_j z + hdot_j into work, in resolve's rhs layouts
  ab2::JacobianRhsArgs ra{adjoint_dims(s), nrhs, dot->stage, dot->term, dot->G0, dot->g0,
                          primal->xs, primal->us, primal->vs, primal->vsT, primal->lam0, primal->lams,
                          work->xs, work->us, work->vs, work->vsT, work->lam0, work->lams};
  CUDA_TRY(ab2::launch_jacobian_rhs(ra, st));
  s->launches += 1;
  // 2. zdot_j = resolve(rho_j) = -K^-1 rho_j
  const ab2_lq_rhs rhs{work->xs, work->us, work->vs, work->vsT, work->lam0, work->lams};
  return run_resolve(s, mueq, mu_dev, nrhs, &rhs, out, st);
}
int ab2_gar_tangent_many(ab2_gar_solver *s, double mueq, int nrhs, const ab2_ls_iterate *primal,
                         const ab2_lq_tangent *dot, const ab2_ls_trial *work, const ab2_ls_trial *out, void *stream) {
  return tangent_many_impl(s, mueq, nullptr, AB2_DEVICE, nrhs, primal, dot, work, out, stream);
}
int ab2_gar_tangent_many_v(ab2_gar_solver *s, const double *mueq, int memspace, int nrhs, const ab2_ls_iterate *primal,
                           const ab2_lq_tangent *dot, const ab2_ls_trial *work, const ab2_ls_trial *out, void *stream) {
  if (!mueq)
    return fail(AB2_ERR_INVALID, "null mueq array");
  return tangent_many_impl(s, 0.0, mueq, memspace, nrhs, primal, dot, work, out, stream);
}

// ---- the generalised streaming kernels (lq_jacobian.cu) as stateless calls: no factorisation, no mu ----
static int check_stateless_handle(const ab2_gar_solver *s, int nrhs, const char *who) {
  if (s->nth > 0 || s->legs > 1)
    return fail(AB2_ERR_UNSUPPORTED, std::string(who) + ": parametric (nth > 0) and parallel handles are not supported");
  if (nrhs < 0)
    return fail(AB2_ERR_INVALID, std::string(who) + ": nrhs < 0");
  return AB2_OK;
}
// the output o may overlap none of the inputs, nor itself
static int refuse_output_overlap(const Fields &o, std::initializer_list<const Fields *> in, const char *who) {
  if (int rc = refuse_overlap(o, o, who))
    return rc;
  for (const Fields *f : in)
    if (int rc = refuse_overlap(o, *f, who))
      return rc;
  return AB2_OK;
}
static ab2::SolVec sol_vec(const ab2_ls_iterate *v, bool each) {
  return v ? ab2::SolVec{v->xs, v->us, v->vs, v->vsT, v->lam0, v->lams, each} : ab2::SolVec{};
}

int ab2_gar_rho_many(ab2_gar_solver *s, int nrhs, int with_vectors, const ab2_lq_tangent *dot1,
                     const ab2_ls_iterate *a1, int a1_each, const ab2_lq_tangent *dot2, const ab2_ls_iterate *a2,
                     int a2_each, const ab2_ls_iterate *e, const ab2_ls_trial *out, void *stream) {
  const char *who = "rho_many";
  if (!s || !dot1 || !a1 || !out || (dot2 && !a2))
    return fail(AB2_ERR_INVALID, "null argument");
  if (int rc = check_stateless_handle(s, nrhs, who))
    return rc;
  const size_t B = s->d.batch, R = (size_t)nrhs * B;
  const bool two = dot2 != nullptr;
  const ab2_lq_tangent none{};
  const ab2_ls_iterate zero{};
  const Fields D1 = rec_fields(s, "dot1", *dot1, R), D2 = rec_fields(s, "dot2", two ? *dot2 : none, R),
               A1 = sol_fields(s, "a1", *a1, a1_each ? R : B), A2 = sol_fields(s, "a2", two ? *a2 : zero, a2_each ? R : B),
               E = sol_fields(s, "e", e ? *e : zero, R), O = sol_fields(s, "out", *out, R);
  for (const Fields *f : {&A1, &O})
    if (int rc = require(*f, who))
      return rc;
  if (two)
    if (int rc = require(A2, who))
      return rc;
  if (e)
    if (int rc = require(E, who))
      return rc;
  if (int rc = refuse_output_overlap(O, {&D1, &D2, &A1, &A2, &E}, who))
    return rc;
  if (nrhs == 0)
    return AB2_OK;
  CUDA_TRY(cudaSetDevice(s->d.device));
  const bool plain = with_vectors && !a1_each && !two && !e;
  ab2::JacobianRhsArgs ra{adjoint_dims(s), nrhs, dot1->stage, dot1->term, dot1->G0, dot1->g0,
                          a1->xs, a1->us, a1->vs, a1->vsT, a1->lam0, a1->lams,
                          out->xs, out->us, out->vs, out->vsT, out->lam0, out->lams};
  if (!plain) {
    ra.ext = true;
    ra.vec = with_vectors != 0;
    ra.z_each = a1_each != 0;
    ra.two = two;
    if (two) {
      ra.stage2 = dot2->stage;
      ra.term2 = dot2->term;
      ra.G02 = dot2->G0;
      ra.z2 = sol_vec(a2, a2_each != 0);
    }
    ra.e = sol_vec(e, true);
  }
  CUDA_TRY(ab2::launch_jacobian_rhs(ra, (cudaStream_t)stream));
  s->launches += 1;
  return AB2_OK;
}

int ab2_gar_grad_many(ab2_gar_solver *s, int nrhs, int with_vectors, const ab2_ls_iterate *y1,
                      const ab2_ls_iterate *z1, int z1_each, const ab2_ls_iterate *y2, const ab2_ls_iterate *z2,
                      int z2_each, const ab2_lq_grad *grad, void *stream) {
  const char *who = "grad_many";
  if (!s || !y1 || !z1 || !grad || (y2 && !z2))
    return fail(AB2_ERR_INVALID, "null argument");
  if (int rc = check_stateless_handle(s, nrhs, who))
    return rc;
  const size_t B = s->d.batch, R = (size_t)nrhs * B;
  const bool two = y2 != nullptr;
  const ab2_ls_iterate zero{};
  const Fields Y1 = sol_fields(s, "y1", *y1, R), Z1 = sol_fields(s, "z1", *z1, z1_each ? R : B),
               Y2 = sol_fields(s, "y2", two ? *y2 : zero, R), Z2 = sol_fields(s, "z2", two ? *z2 : zero, z2_each ? R : B),
               G = rec_fields(s, "grad", *grad, R);
  for (const Fields *f : {&Y1, &Z1, &Y2, &Z2})
    if (int rc = (f == &Y1 || f == &Z1 || two) ? require(*f, who) : AB2_OK)
      return rc;
  if (int rc = refuse_output_overlap(G, {&Y1, &Z1, &Y2, &Z2}, who))
    return rc;
  if (nrhs == 0)
    return AB2_OK;
  CUDA_TRY(cudaSetDevice(s->d.device));
  ab2::JacobianGradArgs ga{adjoint_dims(s), nrhs,
                           z1->xs, z1->us, z1->vs, z1->vsT, z1->lam0, z1->lams,
                           y1->xs, y1->us, y1->vs, y1->vsT, y1->lam0, y1->lams,
                           grad->stage, grad->term, grad->G0, grad->g0, false};
  if (!(with_vectors && !z1_each && !two)) {
    ga.ext = true;
    ga.vec = with_vectors != 0;
    ga.z_each = z1_each != 0;
    ga.y2 = sol_vec(y2, true);
    ga.z2 = sol_vec(z2, z2_each != 0);
  }
  CUDA_TRY(ab2::launch_jacobian_grad(ga, (cudaStream_t)stream));
  s->launches += 1;
  return AB2_OK;
}

// ---- iterative refinement (lq_refine.cu): residual, resolve and update per step, on the last backward's factorisation ----
static bool device_accessible(const void *p) {
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
    cudaGetLastError(); // a plain host pointer on an old runtime: not an error of this call
    return false;
  }
  return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}
// `steps` refinement steps of z against h (own: the problem's own vectors; else rhs), [nrhs][batch][...]; r (in the
// rhs layouts, named like the solution's fields) and dz are the scratch of the residual and the correction.  norms:
// [nrhs][batch][steps + 1] in device or host memory, or null.  The arguments have been checked.
static int run_refine(ab2_gar_solver *s, double mueq, const double *mu_dev, int nrhs, int steps, bool own,
                      const ab2_lq_rhs *rhs, const ab2_ls_trial *z, const ab2_ls_trial *r, const ab2_ls_trial *dz,
                      double *norms, cudaStream_t st) {
  const ab2_gar_dims &d = s->d;
  const int B = d.batch, N = d.horizon;
  const size_t R = (size_t)nrhs * B, nnorm = R * (size_t)(steps + 1);
  Staged nr{nullptr, nullptr, nnorm};
  if (norms) {
    if (int rc = stage_result(s->ref_norms, norms, device_accessible(norms), nnorm, &nr))
      return rc;
    CUDA_TRY(cudaMemsetAsync(nr.dev, 0, nnorm * sizeof(double), st)); // the maxima meet by atomicMax from 0
  }
  auto residual = [&](int col, bool write) -> int {
    ab2::RefineResidualArgs a{};
    a.d = adjoint_dims(s);
    a.nrhs = nrhs;
    a.stage_head = s->p.stage_head;
    a.stage = s->p.stage;
    a.term = s->p.term;
    a.G0 = s->p.G0;
    a.g0 = s->p.g0;
    a.mueq = mueq;
    a.mueq_b = mu_dev;
    a.own = own;
    if (!own) {
      a.hq = rhs->q;
      a.hr = rhs->r;
      a.hd = rhs->d;
      a.hdN = rhs->dN;
      a.hg0 = rhs->g0;
      a.hf = rhs->f;
    }
    a.xs = z->xs;
    a.us = z->us;
    a.vs = z->vs;
    a.vsT = z->vsT;
    a.lam0 = z->lam0;
    a.lams = z->lams;
    if (write) {
      a.q = r->xs;
      a.r = r->us;
      a.dv = r->vs;
      a.dN = r->vsT;
      a.g0out = r->lam0;
      a.f = r->lams;
    }
    a.norms = nr.dev;
    a.nstride = steps + 1;
    a.col = col;
    CUDA_TRY(ab2::launch_refine_residual(a, false, st));
    s->launches += 1;
    return AB2_OK;
  };
  const ab2_lq_rhs rr{r->xs, r->us, r->vs, r->vsT, r->lam0, r->lams};
  // z += dz as a linear step of length 1 over nrhs * batch instances (the [nrhs][batch][...] arrays are contiguous);
  // z + 1.0 * dz rounds to z + dz
  const ab2::LineSearchArgs step{(int)R, N, d.nx, d.nu, d.nc, d.nct, d.nc0,
                                 dz->xs, dz->us, dz->vs, dz->vsT, dz->lam0, dz->lams};
  const ab2::LinearStepIO io{z->xs, z->us, z->vs, z->vsT, z->lam0, z->lams,
                             z->xs, z->us, z->vs, z->vsT, z->lam0, z->lams};
  for (int k = 0; k < steps; ++k) {
    if (int rc = residual(k, true)) // r = K z + h
      return rc;
    if (int rc = run_resolve(s, mueq, mu_dev, nrhs, &rr, dz, st)) // dz = -K^-1 r
      return rc;
    CUDA_TRY(ab2::launch_linear_step(step, io, 1.0, nullptr, st)); // z += dz
    s->launches += 1;
  }
  if (nr.dev) {
    if (int rc = residual(steps, false)) // the last column: the norm of the refined iterate
      return rc;
    return nr.copy_out(st);
  }
  return AB2_OK;
}

// The checks every refinement call shares after the handle's: steps, mu, shared memory.
static int check_refine_args(const ab2_gar_solver *s, double mueq, const double *mueq_arr, int steps, const char *who) {
  if (steps < 0)
    return fail(AB2_ERR_INVALID, std::string(who) + ": steps < 0");
  if (int rc = check_mu(s, mueq, mueq_arr, who))
    return rc;
  return check_resolve_fits(s, who);
}

static int refine_impl(ab2_gar_solver *s, double mueq, const double *mueq_arr, int memspace, int steps, double *norms,
                       void *stream) {
  const char *who = "refine";
  if (!s)
    return fail(AB2_ERR_INVALID, "null solver");
  if (int rc = check_resolve_handle(s, 1, who))
    return rc;
  if (!s->have_primal)
    return fail(AB2_ERR_STATE, std::string(who) + ": the trajectory outputs do not hold the primal solution of the last "
                                                  "backward (no forward since, or an adjoint or tangent call)");
  if (int rc = check_refine_args(s, mueq, mueq_arr, steps, who))
    return rc;
  if (steps == 0 && !norms)
    return AB2_OK;
  cudaStream_t st;
  const double *mu_dev;
  if (int rc = begin_launch(s, mueq_arr, memspace, stream, &st, &mu_dev))
    return rc;
  ab2_ls_trial rdz[2]; // the residual and the correction
  if (int rc = sol_scratch(s, s->ref_buf, 2, rdz))
    return rc;
  const ab2_ls_trial z = trajectory(s);
  return run_refine(s, mueq, mu_dev, 1, steps, true, nullptr, &z, &rdz[0], &rdz[1], norms, st);
}
int ab2_gar_refine(ab2_gar_solver *s, double mueq, int steps, double *norms, void *stream) {
  return refine_impl(s, mueq, nullptr, AB2_DEVICE, steps, norms, stream);
}
int ab2_gar_refine_v(ab2_gar_solver *s, const double *mueq, int memspace, int steps, double *norms, void *stream) {
  if (!mueq)
    return fail(AB2_ERR_INVALID, "null mueq array");
  return refine_impl(s, 0.0, mueq, memspace, steps, norms, stream);
}

static int refine_many_impl(ab2_gar_solver *s, double mueq, const double *mueq_arr, int memspace, int nrhs, int steps,
                            const ab2_lq_rhs *rhs, const ab2_ls_trial *z, const ab2_lq_refine_work *work,
                            double *norms, void *stream) {
  const char *who = "refine_many";
  if (!s || !rhs || !z || !work)
    return fail(AB2_ERR_INVALID, "null argument");
  if (int rc = check_resolve_handle(s, nrhs, who))
    return rc;
  const size_t R = (size_t)nrhs * s->d.batch;
  const Fields H = rhs_fields(s, "rhs", *rhs, R), Z = sol_fields(s, "z", *z, R), WR = rhs_fields(s, "work", *work, R),
               WD = sol_fields(s, "work", *work, R);
  for (const Fields *f : {&Z, &WR, &WD})
    if (int rc = require(*f, who))
      return rc;
  if (int rc = check_refine_args(s, mueq, mueq_arr, steps, who))
    return rc;
  // the residual reads rhs and z and writes work's residual; resolve reads that and writes work's correction; the
  // update reads the correction and writes z, which the next residual reads together with rhs
  for (const FieldPair &ab : {FieldPair{&H, &Z}, FieldPair{&H, &WR}, FieldPair{&H, &WD}, FieldPair{&Z, &Z},
                              FieldPair{&Z, &WR}, FieldPair{&Z, &WD}, FieldPair{&WR, &WR}, FieldPair{&WR, &WD},
                              FieldPair{&WD, &WD}})
    if (int rc = refuse_overlap(*ab.first, *ab.second, who))
      return rc;
  if (nrhs == 0 || (steps == 0 && !norms))
    return AB2_OK;
  cudaStream_t st;
  const double *mu_dev;
  if (int rc = begin_launch(s, mueq_arr, memspace, stream, &st, &mu_dev))
    return rc;
  const ab2_ls_trial r{work->q, work->r, work->d, work->dN, work->g0, work->f};
  const ab2_ls_trial dz{work->xs, work->us, work->vs, work->vsT, work->lam0, work->lams};
  return run_refine(s, mueq, mu_dev, nrhs, steps, false, rhs, z, &r, &dz, norms, st);
}
int ab2_gar_refine_many(ab2_gar_solver *s, double mueq, int nrhs, int steps, const ab2_lq_rhs *rhs,
                        const ab2_ls_trial *z, const ab2_lq_refine_work *work, double *norms, void *stream) {
  return refine_many_impl(s, mueq, nullptr, AB2_DEVICE, nrhs, steps, rhs, z, work, norms, stream);
}
int ab2_gar_refine_many_v(ab2_gar_solver *s, const double *mueq, int memspace, int nrhs, int steps,
                          const ab2_lq_rhs *rhs, const ab2_ls_trial *z, const ab2_lq_refine_work *work, double *norms,
                          void *stream) {
  if (!mueq)
    return fail(AB2_ERR_INVALID, "null mueq array");
  return refine_many_impl(s, 0.0, mueq, memspace, nrhs, steps, rhs, z, work, norms, stream);
}

// the handle's own copy of the records (assemble, sweep_host), allocated on first use
static int own_records(ab2_gar_solver *s) {
  const size_t B = s->d.batch;
  CUDA_TRY(s->own_stage.ensure(stage_total(s)));
  CUDA_TRY(s->own_term.ensure(B * s->trec));
  CUDA_TRY(s->own_G0.ensure(B * s->d.nc0 * s->d.nx));
  CUDA_TRY(s->own_g0.ensure(B * s->d.nc0));
  return AB2_OK;
}

static int assemble_impl(ab2_gar_solver *s, const ab2_lq_inputs *in, const double *preg_b, const double *mu_inv_b,
                         void *stream) {
  if (!s || !in)
    return fail(AB2_ERR_INVALID, "null argument");
  if (s->rec_nth > 0)
    return fail(AB2_ERR_UNSUPPORTED, "assemble: parametric problems (nth > 0) are not supported");
  const ab2_gar_dims &d = s->d;
  const bool stage_ok = d.horizon == 0 || (in->Jx && in->Ju && in->slack && in->Lxx && in->Lxu && in->Luu &&
                                           in->Lx && in->Lu);
  const bool cstr_ok = d.nc == 0 || d.horizon == 0 || (in->cJx && in->cJu && in->Lv && in->shifted && in->lo && in->hi);
  const bool hess_ok = (!in->Hxx && !in->Hxu && !in->Huu) || (in->Hxx && in->Hxu && in->Huu);
  const bool term_ok = in->Lxx_N && in->Lx_N &&
                       (d.nct == 0 || (in->cJx_N && in->Lv_N && in->shifted_N && in->loN && in->hiN));
  const bool init_ok = d.nc0 == 0 || (in->G0 && in->g0);
  if (!stage_ok || !cstr_ok || !hess_ok || !term_ok || !init_ok)
    return fail(AB2_ERR_INVALID, "ab2_lq_inputs: a required array is NULL for these dimensions");
  CUDA_TRY(cudaSetDevice(d.device));
  if (int rc = own_records(s))
    return rc;
  CUDA_TRY(ab2::launch_lq_assemble(*in, preg_b, mu_inv_b, s->own_stage, s->own_term, s->own_G0, s->own_g0, d.batch, d.horizon, d.nx,
                                   d.nu, d.nc, d.nct, d.nc0, s->srec, s->trec, (cudaStream_t)stream));
  s->launches += d.horizon > 0 ? 2 : 1;
  s->p.stage = s->own_stage;
  s->p.stage_head = 0;
  s->p.term = s->own_term;
  s->p.G0 = s->own_G0;
  s->p.g0 = s->own_g0;
  problem_replaced(s, true);
  return AB2_OK;
}
int ab2_gar_assemble(ab2_gar_solver *s, const ab2_lq_inputs *in, void *stream) {
  return assemble_impl(s, in, nullptr, nullptr, stream);
}
int ab2_gar_assemble_v(ab2_gar_solver *s, const ab2_lq_inputs *in, const double *preg, const double *mu_inv, void *stream) {
  if (!preg || !mu_inv)
    return fail(AB2_ERR_INVALID, "assemble_v: null preg / mu_inv array");
  return assemble_impl(s, in, preg, mu_inv, stream);
}

static int copy_ring(const double *base, size_t rec, int knots, int nring, int head, int b0, int nb, int t0, int nt,
                     double *dst, cudaMemcpyKind kind, cudaStream_t st);

// Knots [t0, t0 + nt) of instances [b0, b0 + nb) of a packed VXX, expanded to dense column-major blocks
// [nb][nt][nx*nx] at dst (host: through a stream-ordered device buffer).  head: the factor ring's head.
static int get_vxx_packed(ab2_gar_solver *s, int head, int b0, int nb, int t0, int nt, double *dst, int memspace,
                          cudaStream_t st) {
  const size_t n = (size_t)nb * nt * s->d.nx * s->d.nx;
  if (n == 0)
    return AB2_OK;
  double *out = dst;
  if (memspace != AB2_DEVICE)
    CUDA_TRY(cudaMallocAsync(&out, n * sizeof(double), st));
  ab2::vxx_expand_kernel<<<grid_for(s, n), 256, 0, st>>>(s->out[AB2_OUT_VXX], s->p.Vxx0, out, s->d.horizon, s->d.nx, head,
                                                      b0, nb, t0, nt);
  CUDA_TRY(cudaGetLastError()); // (a copy for the caller, like cudaMemcpy: not in ab2_gar_launch_count)
  if (memspace != AB2_DEVICE) {
    CUDA_TRY(cudaMemcpyAsync(dst, out, n * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaFreeAsync(out, st));
  }
  return AB2_OK;
}

int ab2_gar_problem_ptr(ab2_gar_solver *s, int what, const double **out) {
  if (!s || !out || what < 0 || what > 3)
    return fail(AB2_ERR_INVALID, "bad argument");
  const double *ptrs[4] = {s->p.stage, s->p.term, s->p.G0, s->p.g0};
  *out = ptrs[what];
  return AB2_OK;
}

int ab2_gar_get_problem(ab2_gar_solver *s, int what, double *dst, int memspace, void *stream) {
  if (!s || !dst || what < 0 || what > 3)
    return fail(AB2_ERR_INVALID, "bad argument");
  if (!s->have_problem)
    return fail(AB2_ERR_STATE, "no problem set");
  const double *ptrs[4] = {s->p.stage, s->p.term, s->p.G0, s->p.g0};
  const size_t n[4] = {stage_total(s), (size_t)s->d.batch * s->trec, (size_t)s->d.batch * s->d.nc0 * s->d.nx,
                       (size_t)s->d.batch * s->d.nc0};
  CUDA_TRY(cudaSetDevice(s->d.device));
  if (what == 0 && s->p.stage_head != 0 && n[0]) // the solver-owned copy after cycle_append: knot order through the head
    return copy_ring(s->p.stage, (size_t)s->srec, s->d.horizon, s->d.horizon, s->p.stage_head, 0, s->d.batch, 0,
                     s->d.horizon, dst, out_kind(memspace), (cudaStream_t)stream);
  if (n[what])
    CUDA_TRY(cudaMemcpyAsync(dst, ptrs[what], n[what] * sizeof(double), out_kind(memspace), (cudaStream_t)stream));
  return AB2_OK;
}

// ---- symmetric blocks travel as lower triangles (ab2_gar_sweep_host_sym) ----
namespace ab2 {
// full records from triangle-packed ones: HBM -> HBM, a table look-up per element (built once per CTA)
__global__ void __launch_bounds__(256) expand_sym_kernel(const double *__restrict__ src, double *__restrict__ dst, const long nrec,
                                                         const int nx, const int nu, const int nc, const int srec_full,
                                                         const int srec_pad, const int srec_sym) {
  extern __shared__ int lut[];
  for (int e = threadIdx.x; e < srec_pad; e += blockDim.x)
    lut[e] = e < srec_full ? ab2::sym_source(e, nx, nu, nc) : -1;
  __syncthreads();
  const long total = nrec * srec_pad;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / srec_pad;
    const int e = (int)(i - r * srec_pad), o = lut[e];
    dst[i] = o >= 0 ? src[r * srec_sym + o] : 0.0;
  }
}
} // namespace ab2

size_t ab2_gar_stage_record_doubles_sym(int nx, int nu, int nc) {
  if (nx < 1 || nu < 0 || nc < 0)
    return 0;
  return ab2::stage_sym_len(nx, nu, nc);
}

int ab2_gar_pack_stage_sym(int nx, int nu, int nc, const double *stage, double *stage_sym, long nrec) {
  if (!stage || !stage_sym || nrec < 0 || nx < 1 || nu < 0 || nc < 0)
    return fail(AB2_ERR_INVALID, "bad argument");
  const size_t pad = ab2_gar_stage_record_doubles(nx, nu, nc), sym = ab2_gar_stage_record_doubles_sym(nx, nu, nc);
  // one full-record element per packed slot: the lower-triangle one, which of a symmetric pair has the smaller
  // column-major index and so is written last
  std::vector<int> dst_of(sym, 0);
  for (int e = ab2::stage_offsets(nx, nu, nc).end - 1; e >= 0; --e)
    dst_of[ab2::sym_source(e, nx, nu, nc)] = e;
  for (long k = 0; k < nrec; ++k)
    for (size_t o = 0; o < sym; ++o)
      stage_sym[(size_t)k * sym + o] = stage[(size_t)k * pad + dst_of[o]];
  return AB2_OK;
}

static int sweep_host_impl(ab2_gar_solver *s, const double *stage, const double *term, const double *G0,
                           const double *g0, double mueq, const double *mueq_b, int nchunks, const int *whats,
                           double *const *dsts, int nwhat, void *stream, bool sym);
int ab2_gar_sweep_host(ab2_gar_solver *s, const double *stage, const double *term, const double *G0,
                       const double *g0, double mueq, int nchunks, const int *whats,
                       double *const *dsts, int nwhat, void *stream) {
  return sweep_host_impl(s, stage, term, G0, g0, mueq, nullptr, nchunks, whats, dsts, nwhat, stream, false);
}
int ab2_gar_sweep_host_v(ab2_gar_solver *s, const double *stage, const double *term, const double *G0,
                         const double *g0, const double *mueq, int nchunks, const int *whats,
                         double *const *dsts, int nwhat, void *stream) {
  if (!mueq)
    return fail(AB2_ERR_INVALID, "null mueq array");
  return sweep_host_impl(s, stage, term, G0, g0, 0.0, mueq, nchunks, whats, dsts, nwhat, stream, false);
}
int ab2_gar_sweep_host_sym(ab2_gar_solver *s, const double *stage_sym, const double *term, const double *G0,
                           const double *g0, double mueq, int nchunks, const int *whats,
                           double *const *dsts, int nwhat, void *stream) {
  if (s && (s->rec_nth > 0 || s->legs > 1 || s->dense))
    return fail(AB2_ERR_UNSUPPORTED, "sweep_host_sym: plain (nth = 0) serial handles only");
  return sweep_host_impl(s, stage_sym, term, G0, g0, mueq, nullptr, nchunks, whats, dsts, nwhat, stream, true);
}
int ab2_gar_sweep_host_sym_v(ab2_gar_solver *s, const double *stage_sym, const double *term, const double *G0,
                             const double *g0, const double *mueq, int nchunks, const int *whats,
                             double *const *dsts, int nwhat, void *stream) {
  if (s && (s->rec_nth > 0 || s->legs > 1 || s->dense))
    return fail(AB2_ERR_UNSUPPORTED, "sweep_host_sym: plain (nth = 0) serial handles only");
  if (!mueq)
    return fail(AB2_ERR_INVALID, "null mueq array");
  return sweep_host_impl(s, stage_sym, term, G0, g0, 0.0, mueq, nchunks, whats, dsts, nwhat, stream, true);
}

// mueq_b: per-instance mu in HOST memory (the *_v calls) or null for the scalar mueq
static int sweep_host_impl(ab2_gar_solver *s, const double *stage, const double *term, const double *G0,
                           const double *g0, double mueq, const double *mueq_b, int nchunks, const int *whats,
                           double *const *dsts, int nwhat, void *stream, const bool sym) {
  if (!s || !stage || !term || (s->d.nc0 > 0 && (!G0 || !g0)) || nwhat < 0 || (nwhat > 0 && (!whats || !dsts)))
    return fail(AB2_ERR_INVALID, "bad argument");
  for (int i = 0; i < nwhat; ++i)
    if (whats[i] < 0 || whats[i] >= AB2_OUT_COUNT || !dsts[i])
      return fail(AB2_ERR_INVALID, "bad output selector");
  if (!mueq_b && !(mueq > 0.0) && (s->d.nc > 0 || s->d.nct > 0))
    return fail(AB2_ERR_INVALID, "mueq must be > 0 when constraints are present");
  const double *mu_dev = nullptr; // (staged on the caller's stream, before the fork below)
  if (mueq_b)
    if (int rc = stage_mueq(s, mueq_b, AB2_HOST, (cudaStream_t)stream, &mu_dev))
      return rc;
  CUDA_TRY(cudaSetDevice(s->d.device));
  const int B = s->d.batch, N = s->d.horizon, nx = s->d.nx, nc0 = s->d.nc0;
  constexpr int NS = ab2_gar_solver::kPipeStreams;
  if (!s->pipe_fork) {
    CUDA_TRY(cudaEventCreateWithFlags(&s->pipe_fork, cudaEventDisableTiming));
    for (int i = 0; i < NS; ++i) {
      CUDA_TRY(cudaStreamCreateWithFlags(&s->pipe_stream[i], cudaStreamNonBlocking));
      CUDA_TRY(cudaEventCreateWithFlags(&s->pipe_done[i], cudaEventDisableTiming));
    }
  }
  int rc;
  if ((rc = own_records(s)) != AB2_OK)
    return rc;
  const size_t srec_sym = ab2_gar_stage_record_doubles_sym(nx, s->d.nu, s->d.nc);
  if (sym)
    CUDA_TRY(s->own_stage_sym.ensure((size_t)B * N * srec_sym));
  s->p.stage = s->own_stage;
  s->p.stage_head = 0;
  s->p.term = s->own_term;
  s->p.G0 = s->own_G0;
  s->p.g0 = s->own_g0;
  s->p.do_bwd = 1;
  s->p.do_fwd = 1;
  if (nchunks <= 0) { // enough slices to hide the first upload / last download, each still one full wave
    nchunks = B / 512;
    if (nchunks > 16)
      nchunks = 16;
  }
  if (nchunks < 1)
    nchunks = 1;
  if (nchunks > B)
    nchunks = B;
  cudaStream_t user = (cudaStream_t)stream;
  CUDA_TRY(cudaEventRecord(s->pipe_fork, user));
  for (int i = 0; i < NS && i < nchunks; ++i)
    CUDA_TRY(cudaStreamWaitEvent(s->pipe_stream[i], s->pipe_fork, 0));
  for (int c = 0; c < nchunks; ++c) {
    const int b0 = (int)((long long)B * c / nchunks), b1 = (int)((long long)B * (c + 1) / nchunks);
    const int nb = b1 - b0;
    if (nb <= 0)
      continue;
    cudaStream_t st = s->pipe_stream[c % NS];
    auto up = [&](double *dev, const double *host, size_t per_inst) -> int {
      if (per_inst)
        CUDA_TRY(cudaMemcpyAsync(dev + (size_t)b0 * per_inst, host + (size_t)b0 * per_inst,
                                 (size_t)nb * per_inst * sizeof(double), cudaMemcpyHostToDevice, st));
      return AB2_OK;
    };
    // the small uploads first: enqueued behind the expansion kernel they would sit in the copy engine's queue
    // behind the NEXT slice's records and hold this slice's sweep back by a whole upload
    if ((rc = up(s->own_term, term, s->trec)) != AB2_OK ||
        (rc = up(s->own_G0, G0, (size_t)nc0 * nx)) != AB2_OK || (rc = up(s->own_g0, g0, nc0)) != AB2_OK)
      return rc;
    if (sym) { // lower triangles over PCIe, full records rebuilt in HBM
      if ((rc = up(s->own_stage_sym, stage, (size_t)N * srec_sym)) != AB2_OK)
        return rc;
      const long nrec = (long)nb * N;
      if (nrec > 0) {
        // same shared-memory carve-out as the sweeps it runs beside (an SM is configured for one carve-out at a time)
        static bool carve = false;
        if (!carve) {
          CUDA_TRY(cudaFuncSetAttribute(ab2::expand_sym_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                        (int)cudaSharedmemCarveoutMaxShared));
          carve = true;
        }
        if (s->srec * sizeof(int) > 48 * 1024) // (records beyond 12 288 doubles: opt in to the larger table)
          CUDA_TRY(cudaFuncSetAttribute(ab2::expand_sym_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)(s->srec * sizeof(int))));
        ab2::expand_sym_kernel<<<grid_for(s, (size_t)nrec * s->srec), 256, s->srec * sizeof(int), st>>>(
            s->own_stage_sym + (size_t)b0 * N * srec_sym, s->own_stage + (size_t)b0 * N * s->srec, nrec, nx, s->d.nu, s->d.nc,
            ab2::stage_offsets(nx, s->d.nu, s->d.nc).end, (int)s->srec, (int)srec_sym);
        CUDA_TRY(cudaGetLastError());
        s->launches += 1;
      }
    } else if ((rc = up(s->own_stage, stage, (size_t)N * s->srec)) != AB2_OK)
      return rc;
    ab2::SweepParams q = slice_params(s, b0, nb);
    if (mu_dev)
      q.mueq_b = mu_dev + b0;
    else
      q.mueq = mueq;
    if (int rc2 = run_kernels(s, q, 1, 1, st))
      return rc2;
    for (int i = 0; i < nwhat; ++i) {
      const int w = whats[i];
      const size_t per_inst = (size_t)s->out_knots[w] * s->out_rec[w];
      if (w == AB2_OUT_VXX && warp_kernel(s)) {
        if ((rc = get_vxx_packed(s, 0, b0, nb, 0, N + 1, dsts[i] + (size_t)b0 * per_inst, AB2_HOST, st)) != AB2_OK)
          return rc;
      } else if (per_inst)
        CUDA_TRY(cudaMemcpyAsync(dsts[i] + (size_t)b0 * per_inst, s->out[w] + (size_t)b0 * per_inst,
                                 (size_t)nb * per_inst * sizeof(double), cudaMemcpyDeviceToHost, st));
    }
  }
  for (int i = 0; i < NS && i < nchunks; ++i) {
    CUDA_TRY(cudaEventRecord(s->pipe_done[i], s->pipe_stream[i]));
    CUDA_TRY(cudaStreamWaitEvent(user, s->pipe_done[i], 0));
  }
  swept_host(s, mueq, mu_dev);
  return AB2_OK;
}

size_t ab2_gar_output_doubles(const ab2_gar_solver *s, int what) {
  if (!s || what < 0 || what >= AB2_OUT_COUNT)
    return 0;
  return s->out_doubles[what];
}

// Dense copy of knots [t0, t0 + nt) of instances [b0, b0 + nb) of a per-knot array whose first `nring` knots
// are ring-indexed with head `head` (knot t in slot (t + head) mod nring; knots >= nring -- the terminal
// entry of VXX / VX -- stay in place): at most three strided copies.
static int copy_ring(const double *base, size_t rec, int knots, int nring, int head, int b0, int nb, int t0, int nt,
                     double *dst, cudaMemcpyKind kind, cudaStream_t st) {
  auto piece = [&](int lt, int pt, int len) -> int { // logical start, physical start, length
    if (len <= 0)
      return AB2_OK;
    CUDA_TRY(cudaMemcpy2DAsync(dst + (size_t)(lt - t0) * rec, (size_t)nt * rec * sizeof(double),
                               base + ((size_t)b0 * knots + pt) * rec, (size_t)knots * rec * sizeof(double),
                               (size_t)len * rec * sizeof(double), (size_t)nb, kind, st));
    return AB2_OK;
  };
  const int t1 = t0 + nt;
  auto clip = [&](int lo, int hi, int shift) { // logical [lo, hi) of the ring, physical = logical + shift
    const int a = t0 > lo ? t0 : lo, b = t1 < hi ? t1 : hi;
    return piece(a, a + shift, b - a);
  };
  int rc;
  if ((rc = clip(0, nring - head, head)) != AB2_OK || (rc = clip(nring - head, nring, head - nring)) != AB2_OK ||
      (rc = clip(nring, knots, 0)) != AB2_OK)
    return rc;
  return AB2_OK;
}
static bool ring_indexed(const ab2_gar_solver *s, int what) {
  return s->fac_head != 0 && (what == AB2_OUT_FF || what == AB2_OUT_FB || what == AB2_OUT_VXX || what == AB2_OUT_VX);
}

int ab2_gar_get(ab2_gar_solver *s, int what, double *dst, int memspace, void *stream) {
  if (!s || !dst || what < 0 || what >= AB2_OUT_COUNT)
    return fail(AB2_ERR_INVALID, "bad argument");
  CUDA_TRY(cudaSetDevice(s->d.device));
  if (s->out_doubles[what] == 0)
    return AB2_OK;
  if (what == AB2_OUT_VXX && s->vxx_packed)
    return get_vxx_packed(s, s->fac_head, 0, s->d.batch, 0, s->d.horizon + 1, dst, memspace, (cudaStream_t)stream);
  if (ring_indexed(s, what)) // between a cycle_append and the next backward: knot order through the ring head
    return copy_ring(s->out[what], s->out_rec[what], s->out_knots[what], s->d.horizon, s->fac_head, 0, s->d.batch, 0,
                     s->out_knots[what], dst, out_kind(memspace), (cudaStream_t)stream);
  CUDA_TRY(cudaMemcpyAsync(dst, s->out[what], s->out_doubles[what] * sizeof(double), out_kind(memspace),
                           (cudaStream_t)stream));
  return AB2_OK;
}

int ab2_gar_get_range(ab2_gar_solver *s, int what, int b0, int nb, int t0, int nt, double *dst,
                      int memspace, void *stream) {
  if (!s || !dst || what < 0 || what >= AB2_OUT_COUNT)
    return fail(AB2_ERR_INVALID, "bad argument");
  const int knots = s->out_knots[what];
  if (b0 < 0 || nb < 0 || b0 + nb > s->d.batch || t0 < 0 || nt < 0 || t0 + nt > knots)
    return fail(AB2_ERR_INVALID, "range out of bounds");
  CUDA_TRY(cudaSetDevice(s->d.device));
  const size_t rec = s->out_rec[what];
  if (rec == 0 || nb == 0 || nt == 0)
    return AB2_OK;
  if (what == AB2_OUT_VXX && s->vxx_packed)
    return get_vxx_packed(s, s->fac_head, b0, nb, t0, nt, dst, memspace, (cudaStream_t)stream);
  if (ring_indexed(s, what))
    return copy_ring(s->out[what], rec, knots, s->d.horizon, s->fac_head, b0, nb, t0, nt, dst, out_kind(memspace),
                     (cudaStream_t)stream);
  const double *src = s->out[what] + ((size_t)b0 * knots + t0) * rec;
  CUDA_TRY(cudaMemcpy2DAsync(dst, (size_t)nt * rec * sizeof(double), src, (size_t)knots * rec * sizeof(double),
                             (size_t)nt * rec * sizeof(double), (size_t)nb, out_kind(memspace), (cudaStream_t)stream));
  return AB2_OK;
}

int ab2_gar_first_step_policy(ab2_gar_solver *s, double *dst, void *stream) {
  if (!s || !dst)
    return fail(AB2_ERR_INVALID, "bad argument");
  if (s->d.horizon < 1)
    return fail(AB2_ERR_INVALID, "first_step_policy needs horizon >= 1");
  if (s->dense)
    return fail(AB2_ERR_UNSUPPORTED, "first_step_policy: not offered by the stage-dense solver");
  if (!s->have_backward)
    return fail(AB2_ERR_STATE, "first_step_policy before backward()");
  CUDA_TRY(cudaSetDevice(s->d.device));
  const size_t total = (size_t)s->d.batch * s->d.nu * (s->d.nx + 1);
  ab2::first_step_policy_kernel<<<grid_for(s, total), 256, 0, (cudaStream_t)stream>>>(
      s->out[AB2_OUT_FB], s->out[AB2_OUT_FF], dst, s->d.batch, s->d.horizon, s->nr, s->d.nu, s->d.nx, s->fac_head);
  CUDA_TRY(cudaGetLastError());
  s->launches += 1;
  return AB2_OK;
}

int ab2_gar_get_gains(ab2_gar_solver *s, double *dst, int memspace, void *stream) {
  if (!s || !dst)
    return fail(AB2_ERR_INVALID, "bad argument");
  if (!s->have_backward)
    return fail(AB2_ERR_STATE, "get_gains before backward()");
  if (s->dense)
    return fail(AB2_ERR_UNSUPPORTED, "get_gains: the results_.gains_ layout is the proximal solver's");
  CUDA_TRY(cudaSetDevice(s->d.device));
  const long nrec = (long)s->d.batch * s->d.horizon;
  const size_t total = (size_t)nrec * s->nr * (s->d.nx + 1);
  if (total == 0)
    return AB2_OK;
  Staged r;
  if (int rc = stage_result(s->gains_tmp, dst, memspace == AB2_DEVICE, total, &r))
    return rc;
  ab2::gains_kernel<<<grid_for(s, total), 256, 0, (cudaStream_t)stream>>>(s->out[AB2_OUT_FB], s->out[AB2_OUT_FF], r.dev,
                                                                          nrec, s->nr, s->d.nx, s->d.horizon, s->fac_head);
  CUDA_TRY(cudaGetLastError());
  s->launches += 1;
  return r.copy_out((cudaStream_t)stream);
}

static int kkt_error_impl(ab2_gar_solver *s, double mueq, const double *mueq_b, double *dst, int memspace, void *stream) {
  if (!s || !dst)
    return fail(AB2_ERR_INVALID, "bad argument");
  if (!s->have_problem || !s->have_backward || !s->have_forward)
    return fail(AB2_ERR_STATE, "kkt_error needs a problem and a completed sweep (no forward pass since the last backward)");
  if (s->rec_nth > 0)
    return fail(AB2_ERR_UNSUPPORTED, "kkt_error: parametric problems (nth > 0) are not supported");
  CUDA_TRY(cudaSetDevice(s->d.device));
  Staged r;
  if (int rc = stage_result(s->kkt_tmp, dst, memspace == AB2_DEVICE, (size_t)s->d.batch * 3, &r))
    return rc;
  // the refinement's residual of the last forward pass against the problem's own vectors, with one norm per row family
  ab2::RefineResidualArgs a{};
  a.d = adjoint_dims(s);
  a.nrhs = 1;
  a.stage_head = s->p.stage_head;
  a.stage = s->p.stage;
  a.term = s->p.term;
  a.G0 = s->p.G0;
  a.g0 = s->p.g0;
  a.mueq = mueq;
  a.mueq_b = mueq_b;
  a.own = true;
  const ab2_ls_trial z = trajectory(s);
  a.xs = z.xs;
  a.us = z.us;
  a.vs = z.vs;
  a.vsT = z.vsT;
  a.lam0 = z.lam0;
  a.lams = z.lams;
  a.norms = r.dev;
  a.nstride = 3;
  a.col = 0;
  CUDA_TRY(cudaMemsetAsync(a.norms, 0, r.n * sizeof(double), (cudaStream_t)stream));
  CUDA_TRY(ab2::launch_refine_residual(a, true, (cudaStream_t)stream));
  s->launches += 1;
  return r.copy_out((cudaStream_t)stream);
}
int ab2_gar_kkt_error(ab2_gar_solver *s, double mueq, double *dst, int memspace, void *stream) {
  return kkt_error_impl(s, mueq, nullptr, dst, memspace, stream);
}
int ab2_gar_kkt_error_v(ab2_gar_solver *s, const double *mueq, double *dst, int memspace, void *stream) {
  if (!mueq)
    return fail(AB2_ERR_INVALID, "null mueq array");
  return kkt_error_impl(s, 0.0, mueq, dst, memspace, stream);
}

int ab2_gar_device_ptr(ab2_gar_solver *s, int what, double **out) {
  if (!s || !out || what < 0 || what >= AB2_OUT_COUNT)
    return fail(AB2_ERR_INVALID, "bad argument");
  *out = s->out[what];
  return AB2_OK;
}

int ab2_gar_status(ab2_gar_solver *s, int *dst, int memspace, void *stream) {
  if (!s || !dst)
    return fail(AB2_ERR_INVALID, "bad argument");
  CUDA_TRY(cudaSetDevice(s->d.device));
  CUDA_TRY(cudaMemcpyAsync(dst, s->status, sizeof(int) * s->d.batch, out_kind(memspace), (cudaStream_t)stream));
  return AB2_OK;
}

// ---- line-search consumers (linesearch.cu) ----
static ab2::LineSearchArgs ls_args(const ab2_gar_solver *s) {
  ab2::LineSearchArgs a;
  a.batch = s->d.batch;
  a.N = s->d.horizon;
  a.nx = s->d.nx;
  a.nu = s->d.nu;
  a.nc = s->d.nc;
  a.nct = s->d.nct;
  a.nc0 = s->d.nc0;
  const ab2_ls_trial z = trajectory(s);
  a.dxs = z.xs;
  a.dus = z.us;
  a.dvs = z.vs;
  a.dvsT = z.vsT;
  a.dlam0 = z.lam0;
  a.dlams = z.lams;
  return a;
}
static int linear_step_impl(ab2_gar_solver *s, double alpha, const double *alpha_b, const ab2_ls_iterate *cur,
                            const ab2_ls_trial *trial, void *stream) {
  if (!s || !cur || !trial)
    return fail(AB2_ERR_INVALID, "null argument");
  if (!s->have_forward)
    return fail(AB2_ERR_STATE, "linear_step needs the step of a forward pass");
  const ab2_gar_dims &d = s->d;
  const bool ok = cur->xs && trial->xs && (d.horizon == 0 || (cur->us && trial->us && cur->lams && trial->lams)) &&
                  (d.nc == 0 || d.horizon == 0 || (cur->vs && trial->vs)) && (d.nct == 0 || (cur->vsT && trial->vsT)) &&
                  (d.nc0 == 0 || (cur->lam0 && trial->lam0));
  if (!ok)
    return fail(AB2_ERR_INVALID, "linear_step: a required array is NULL for these dimensions");
  CUDA_TRY(cudaSetDevice(d.device));
  ab2::LinearStepIO io{cur->xs, cur->us, cur->vs, cur->vsT, cur->lam0, cur->lams,
                       trial->xs, trial->us, trial->vs, trial->vsT, trial->lam0, trial->lams};
  CUDA_TRY(ab2::launch_linear_step(ls_args(s), io, alpha, alpha_b, (cudaStream_t)stream));
  s->launches += 1;
  return AB2_OK;
}
int ab2_gar_linear_step(ab2_gar_solver *s, double alpha, const ab2_ls_iterate *cur, const ab2_ls_trial *trial,
                        void *stream) {
  return linear_step_impl(s, alpha, nullptr, cur, trial, stream);
}
int ab2_gar_linear_step_v(ab2_gar_solver *s, const double *alpha, const ab2_ls_iterate *cur, const ab2_ls_trial *trial,
                          void *stream) {
  if (!alpha)
    return fail(AB2_ERR_INVALID, "null alpha array");
  return linear_step_impl(s, 0.0, alpha, cur, trial, stream);
}
int ab2_gar_directional_derivative(ab2_gar_solver *s, const double *Lxs, const double *Lus, double *dst, int memspace,
                                   void *stream) {
  if (!s || !Lxs || !dst || (s->d.horizon > 0 && !Lus))
    return fail(AB2_ERR_INVALID, "null argument");
  if (!s->have_forward)
    return fail(AB2_ERR_STATE, "directional_derivative needs the step of a forward pass");
  CUDA_TRY(cudaSetDevice(s->d.device));
  Staged r;
  if (int rc = stage_result(s->ls_tmp, dst, memspace == AB2_DEVICE, s->d.batch, &r))
    return rc;
  CUDA_TRY(ab2::launch_directional_derivative(ls_args(s), Lxs, Lus, r.dev, (cudaStream_t)stream));
  s->launches += 1;
  return r.copy_out((cudaStream_t)stream);
}
static int al_value_impl(ab2_gar_solver *s, const ab2_ls_iterate *plus, const double *cost, double mudyn, double mucstr,
                         const double *mudyn_b, const double *mucstr_b, double *dst, int memspace, void *stream) {
  if (!s || !plus || !dst)
    return fail(AB2_ERR_INVALID, "null argument");
  const ab2_gar_dims &d = s->d;
  if ((d.nc0 > 0 && !plus->lam0) || (d.horizon > 0 && !plus->lams) || (d.nc > 0 && d.horizon > 0 && !plus->vs) ||
      (d.nct > 0 && !plus->vsT))
    return fail(AB2_ERR_INVALID, "al_value: a required multiplier array is NULL for these dimensions");
  CUDA_TRY(cudaSetDevice(d.device));
  Staged r;
  if (int rc = stage_result(s->ls_tmp, dst, memspace == AB2_DEVICE, d.batch, &r))
    return rc;
  CUDA_TRY(ab2::launch_al_value(d.batch, d.horizon, d.nx, d.nc, d.nct, d.nc0, plus->lam0, plus->lams, plus->vs, plus->vsT,
                                cost, mudyn, mucstr, mudyn_b, mucstr_b, r.dev, (cudaStream_t)stream));
  s->launches += 1;
  return r.copy_out((cudaStream_t)stream);
}
int ab2_gar_al_value(ab2_gar_solver *s, const ab2_ls_iterate *plus, const double *cost, double mudyn, double mucstr,
                     double *dst, int memspace, void *stream) {
  return al_value_impl(s, plus, cost, mudyn, mucstr, nullptr, nullptr, dst, memspace, stream);
}
int ab2_gar_al_value_v(ab2_gar_solver *s, const ab2_ls_iterate *plus, const double *cost, const double *mudyn,
                       const double *mucstr, double *dst, int memspace, void *stream) {
  if (!mudyn || !mucstr)
    return fail(AB2_ERR_INVALID, "al_value_v: null mudyn / mucstr array");
  return al_value_impl(s, plus, cost, 0.0, 0.0, mudyn, mucstr, dst, memspace, stream);
}

// ---- multipliers, Lagrangian gradient, criterion (proxddp_inner.cu) ----
static ab2::InnerDims inner_dims(const ab2_gar_solver *s) {
  const ab2_gar_dims &d = s->d;
  return ab2::InnerDims{d.batch, d.horizon, d.nx, d.nu, d.nc, d.nct, d.nc0};
}
static int multipliers_impl(ab2_gar_solver *s, const ab2_mult_inputs *in, const double *mu_b, const double *mu_dyn_b,
                            const ab2_mult_outputs *out, double *dst, int memspace, void *stream) {
  if (!s || !in || !out || !dst)
    return fail(AB2_ERR_INVALID, "null argument");
  const ab2_gar_dims &d = s->d;
  const bool stages = d.horizon > 0;
  if (stages && (in->xnext != nullptr) == (in->fs != nullptr))
    return fail(AB2_ERR_INVALID, "multipliers: give exactly one of xnext and fs");
  const bool ok = (!stages || ((in->fs || in->xs) && in->lams && out->slack && out->lams_plus)) &&
                  (d.nc0 == 0 || (in->init_value && in->lam0 && out->lam0_plus)) &&
                  (d.nc == 0 || !stages ||
                   (in->vs && in->prev_vs && in->cval && in->lo && in->hi && out->vs_plus && out->shifted && out->Lv)) &&
                  (d.nct == 0 || (in->vsT && in->prev_vsT && in->cval_N && in->loN && in->hiN && out->vsT_plus &&
                                  out->shifted_N && out->Lv_N));
  if (!ok)
    return fail(AB2_ERR_INVALID, "multipliers: a required array is NULL for these dimensions");
  if (!mu_b && (!(in->mu > 0.0) || !(in->mu_dyn > 0.0)))
    return fail(AB2_ERR_INVALID, "multipliers: mu and mu_dyn must be positive");
  CUDA_TRY(cudaSetDevice(d.device));
  Staged r;
  if (int rc = stage_result(s->inner_tmp, dst, memspace == AB2_DEVICE, (size_t)d.batch * 2, &r))
    return rc;
  CUDA_TRY(ab2::launch_multipliers(inner_dims(s), *in, mu_b, mu_dyn_b, *out, r.dev, (cudaStream_t)stream));
  s->launches += 1;
  return r.copy_out((cudaStream_t)stream);
}
int ab2_gar_multipliers(ab2_gar_solver *s, const ab2_mult_inputs *in, const ab2_mult_outputs *out, double *dst,
                        int memspace, void *stream) {
  return multipliers_impl(s, in, nullptr, nullptr, out, dst, memspace, stream);
}
int ab2_gar_multipliers_v(ab2_gar_solver *s, const ab2_mult_inputs *in, const double *mu, const double *mu_dyn,
                          const ab2_mult_outputs *out, double *dst, int memspace, void *stream) {
  if (!mu || !mu_dyn)
    return fail(AB2_ERR_INVALID, "multipliers_v: null mu / mu_dyn array");
  return multipliers_impl(s, in, mu, mu_dyn, out, dst, memspace, stream);
}
int ab2_gar_lagrangian_gradient(ab2_gar_solver *s, const ab2_lag_inputs *in, const ab2_lag_outputs *out, void *stream) {
  if (!s || !in || !out)
    return fail(AB2_ERR_INVALID, "null argument");
  const ab2_gar_dims &d = s->d;
  const bool stages = d.horizon > 0;
  if (!out->Lx && !out->Lx_N && !out->Lu && !out->Lxs && !out->Lus)
    return fail(AB2_ERR_INVALID, "lagrangian_gradient: no output array given");
  const bool ok = in->lx_N && (!stages || (in->lx && in->lu && in->Jx && in->Ju && in->lams)) &&
                  (d.nc == 0 || !stages || (in->cJx && in->cJu && in->vs)) && (d.nct == 0 || (in->cJx_N && in->vsT)) &&
                  (d.nc0 == 0 || (in->G0 && in->lam0));
  if (!ok)
    return fail(AB2_ERR_INVALID, "lagrangian_gradient: a required input array is NULL for these dimensions");
  CUDA_TRY(cudaSetDevice(d.device));
  CUDA_TRY(ab2::launch_lagrangian_gradient(inner_dims(s), *in, *out, (cudaStream_t)stream));
  s->launches += 1;
  return AB2_OK;
}
int ab2_gar_criterion(ab2_gar_solver *s, const double *Lxs, const double *Lus, const double *init_value,
                      const double *slack, const double *Lv, const double *Lv_N, double *dst, int memspace,
                      void *stream) {
  if (!s || !dst)
    return fail(AB2_ERR_INVALID, "null argument");
  const ab2_gar_dims &d = s->d;
  const bool stages = d.horizon > 0;
  const bool ok = Lxs && (!stages || Lus) && (d.nc0 == 0 || !stages || init_value) && (d.horizon < 2 || slack) &&
                  (d.nc == 0 || !stages || Lv) && (d.nct == 0 || Lv_N);
  if (!ok)
    return fail(AB2_ERR_INVALID, "criterion: a required array is NULL for these dimensions");
  CUDA_TRY(cudaSetDevice(d.device));
  Staged r;
  if (int rc = stage_result(s->inner_tmp, dst, memspace == AB2_DEVICE, (size_t)d.batch * 2, &r))
    return rc;
  CUDA_TRY(ab2::launch_criterion(inner_dims(s), Lxs, Lus, init_value, slack, Lv, Lv_N, r.dev, (cudaStream_t)stream));
  s->launches += 1;
  return r.copy_out((cudaStream_t)stream);
}

static int fddp_backward_impl(ab2_gar_solver *s, const ab2_fddp_inputs *in, const double *preg_b, double *Vx_out,
                              double *Quuks_out, void *stream) {
  if (!s || !in)
    return fail(AB2_ERR_INVALID, "null argument");
  const ab2_gar_dims &d = s->d;
  if (d.nc != 0 || d.nct != 0 || d.nc0 != d.nx || s->rec_nth != 0 || s->legs > 1 || d.horizon < 1)
    return fail(AB2_ERR_INVALID, "fddp_backward_pass needs a serial solver with nc = nct = 0, nc0 = nx, horizon >= 1");
  if (!in->Jx || !in->Ju || !in->fs || !in->Lxx || !in->Lxu || !in->Luu || !in->Lx || !in->Lu || !in->Lxx_N || !in->Lx_N)
    return fail(AB2_ERR_INVALID, "ab2_fddp_inputs: a required array is NULL");
  CUDA_TRY(cudaSetDevice(d.device));
  cudaStream_t st = (cudaStream_t)stream;
  const int B = d.batch, N = d.horizon, nx = d.nx, nu = d.nu;
  CUDA_TRY(s->fddp_slack.ensure((size_t)B * N * nx));
  CUDA_TRY(s->fddp_G0.ensure((size_t)B * nx * nx));
  CUDA_TRY(s->fddp_g0.ensure((size_t)B * nx));
  CUDA_TRY(s->fddp_vx.ensure((size_t)B * (N + 1) * nx));
  ab2::fddp_prep_kernel<<<s->p.num_sms * 4, 256, 0, st>>>(in->fs, s->fddp_slack, s->fddp_G0, s->fddp_g0, B, N, nx);
  CUDA_TRY(cudaGetLastError());
  s->launches += 1;
  ab2_lq_inputs lq;
  std::memset(&lq, 0, sizeof(lq));
  lq.Jx = in->Jx;
  lq.Ju = in->Ju;
  lq.slack = s->fddp_slack;
  lq.Lxx = in->Lxx;
  lq.Lxu = in->Lxu;
  lq.Luu = in->Luu;
  lq.Lx = in->Lx;
  lq.Lu = in->Lu;
  lq.Lxx_N = in->Lxx_N;
  lq.Lx_N = in->Lx_N;
  lq.G0 = s->fddp_G0;
  lq.g0 = s->fddp_g0;
  lq.preg = in->preg; // Q, R and the terminal Q carry + preg I (:217, :246, :273)
  lq.mu_inv = 1.0;
  if (int rc = assemble_impl(s, &lq, preg_b, nullptr, stream))
    return rc;
  if (int rc = ab2_gar_backward(s, 1.0, stream)) // (mueq is unused without constraints)
    return rc;
  double *vxo = Vx_out ? Vx_out : s->fddp_vx.p;
  ab2::fddp_vx_kernel<<<s->p.num_sms * 4, 256, 0, st>>>(s->out[AB2_OUT_VXX], s->vxx_packed ? s->p.Vxx0 : nullptr,
                                                      s->out[AB2_OUT_VX], in->fs, vxo, B, N, nx);
  CUDA_TRY(cudaGetLastError());
  s->launches += 1;
  if (Quuks_out) {
    ab2::fddp_quuks_kernel<<<s->p.num_sms * 4, 256, 0, st>>>(in->Ju, in->Lu, vxo, Quuks_out, B, N, nx, nu);
    CUDA_TRY(cudaGetLastError());
    s->launches += 1;
  }
  return AB2_OK;
}
int ab2_fddp_backward_pass(ab2_gar_solver *s, const ab2_fddp_inputs *in, double *Vx_out, double *Quuks_out, void *stream) {
  return fddp_backward_impl(s, in, nullptr, Vx_out, Quuks_out, stream);
}
int ab2_fddp_backward_pass_v(ab2_gar_solver *s, const ab2_fddp_inputs *in, const double *preg, double *Vx_out,
                             double *Quuks_out, void *stream) {
  if (!preg)
    return fail(AB2_ERR_INVALID, "fddp_backward_pass_v: null preg array");
  return fddp_backward_impl(s, in, preg, Vx_out, Quuks_out, stream);
}

int ab2_gar_collapse_feedback(ab2_gar_solver *s, void *stream) {
  if (!s)
    return fail(AB2_ERR_INVALID, "null solver");
  if (s->legs <= 1)
    return AB2_OK; // the serial solver's collapseFeedback is a no-op (riccati-base.hpp:32)
  if (!s->have_backward)
    return fail(AB2_ERR_STATE, "collapse_feedback before backward()");
  if (s->d.horizon < 1)
    return AB2_OK;
  CUDA_TRY(cudaSetDevice(s->d.device));
  CUDA_TRY(ab2::launch_collapse(s->p, s->d.nx, s->d.nu, s->d.nc, (cudaStream_t)stream));
  s->launches += 1;
  return AB2_OK;
}

int ab2_gar_pivot_stats(ab2_gar_solver *s, int *dst, int memspace, void *stream) {
  if (!s || !dst)
    return fail(AB2_ERR_INVALID, "bad argument");
  if (!s->have_backward)
    return fail(AB2_ERR_STATE, "pivot_stats before backward()");
  CUDA_TRY(cudaSetDevice(s->d.device));
  CUDA_TRY(cudaMemcpyAsync(dst, s->pivstat, sizeof(int) * s->d.batch, out_kind(memspace), (cudaStream_t)stream));
  return AB2_OK;
}

int ab2_gar_cycle_append(ab2_gar_solver *s, const double *new_last, int memspace, void *stream) {
  if (!s || !new_last)
    return fail(AB2_ERR_INVALID, "bad argument");
  const int N = s->d.horizon, B = s->d.batch;
  if (N < 1)
    return fail(AB2_ERR_INVALID, "cycle_append needs horizon >= 1");
  if (s->rec_nth > 0)
    return fail(AB2_ERR_UNSUPPORTED, "cycle_append: parametric problems (nth > 0) are not supported");
  CUDA_TRY(cudaSetDevice(s->d.device));
  cudaStream_t st = (cudaStream_t)stream;
  // factors: datas[0..N-1] rotate left, datas[N-1] re-created (zeros), terminal kept
  // (proximal-riccati.hxx:79-83).  Vxx/vx have N+1 entries; the last is the terminal's.
  if (s->legs > 1) { // the parallel solver drops every factor and starts over (parallel-solver.hxx:246-258)
    for (int w : {AB2_OUT_FF, AB2_OUT_FB, AB2_OUT_VXX, AB2_OUT_VX, AB2_OUT_FTH, AB2_OUT_VXT, AB2_OUT_VTT, AB2_OUT_VT})
      if (s->out_doubles[w])
        CUDA_TRY(cudaMemsetAsync(s->out[w], 0, s->out_doubles[w] * sizeof(double), st));
  }
  // O(1) in the horizon: nothing moves.  The per-knot factor arrays and the solver-owned stage records are rings;
  // rotating left = advancing the head by one.  What is touched is ONE knot slot per instance and array:
  // the factor slot of the new last knot is zeroed (datas[N-1] re-created, :82-83), its record is written.
  if (s->legs <= 1) {
    const int slot = s->fac_head; // the old knot 0's slot, which holds the new stage knot N-1 once cycled() has
                                  // advanced the head by one
    for (int w : {AB2_OUT_FF, AB2_OUT_FB, AB2_OUT_VXX, AB2_OUT_VX}) {
      const size_t rec = (w == AB2_OUT_VXX && s->vxx_packed) ? (size_t)ab2::vxx_packed_doubles(s->d.nx) : s->out_rec[w];
      if (rec == 0)
        continue;
      CUDA_TRY(cudaMemset2DAsync(s->out[w] + (size_t)slot * rec, (size_t)s->out_knots[w] * rec * sizeof(double), 0,
                                 rec * sizeof(double), (size_t)B, st));
    }
    if (s->vxx_packed && ab2::vxx_slot_is_full(slot)) // slot 0's block lives in the full array
      CUDA_TRY(cudaMemsetAsync(s->p.Vxx0, 0, (size_t)B * s->d.nx * s->d.nx * sizeof(double), st));
  }
  // kkt0 zeroed (:84-86)
  if (s->out_doubles[AB2_OUT_KKT0])
    CUDA_TRY(cudaMemsetAsync(s->out[AB2_OUT_KKT0], 0, s->out_doubles[AB2_OUT_KKT0] * sizeof(double), st));
  // the problem itself: our own device copy (host-fed problems) rotates the same way; a device-resident
  // caller rotates its own buffers, like cycleProblem does for the reference's problem (solver-proxddp.hxx:202-209).
  if (s->own_stage && s->p.stage == s->own_stage) {
    s->p.stage_head = (s->p.stage_head + 1) % N;
    const int slot = (N - 1 + s->p.stage_head) % N;
    CUDA_TRY(cudaMemcpy2DAsync(s->own_stage + (size_t)slot * s->srec, (size_t)N * s->srec * sizeof(double),
                               new_last, (size_t)s->srec * sizeof(double), (size_t)s->srec * sizeof(double),
                               (size_t)B,
                               memspace == AB2_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
  }
  CUDA_TRY(cudaGetLastError());
  cycled(s);
  return AB2_OK;
}

int ab2_gar_phase_clocks(ab2_gar_solver *s, long long *dst16) { // AB2_PHASE_CLOCKS=1: cycles per phase, instance 0
  if (!s || !dst16 || !s->p.clk)
    return fail(AB2_ERR_STATE, "phase clocks are off (set AB2_PHASE_CLOCKS=1 before create)");
  CUDA_TRY(cudaMemcpy(dst16, s->p.clk, 16 * sizeof(long long), cudaMemcpyDeviceToHost));
  CUDA_TRY(cudaMemset(s->p.clk, 0, 16 * sizeof(long long)));
  return AB2_OK;
}

int ab2_gar_ring_heads(const ab2_gar_solver *s, int *factor_head, int *stage_head) {
  if (!s)
    return fail(AB2_ERR_INVALID, "null solver");
  if (factor_head)
    *factor_head = s->fac_head;
  if (stage_head)
    *stage_head = s->p.stage_head;
  return AB2_OK;
}

int ab2_gar_synchronize(ab2_gar_solver *s, void *stream) {
  if (!s)
    return fail(AB2_ERR_INVALID, "null solver");
  CUDA_TRY(cudaSetDevice(s->d.device));
  CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));
  return AB2_OK;
}

// ---- multi-GPU: fused pack + all-gather of the first-step policy over NVLink peer memory ----
int ab2_gar_peer_gather_init(ab2_gar_solver *s, int world, int rank, void *ipc_handle_out) {
  if (!s || !ipc_handle_out || world < 1 || world > ab2::kMaxPeers || rank < 0 || rank >= world)
    return fail(AB2_ERR_INVALID, "peer_gather_init: bad argument (world <= 8)");
  if (s->d.horizon < 1)
    return fail(AB2_ERR_INVALID, "peer_gather needs horizon >= 1");
  if (s->pg_local)
    return fail(AB2_ERR_STATE, "peer_gather_init called twice");
  CUDA_TRY(cudaSetDevice(s->d.device));
  const size_t per = (size_t)s->d.nu * (s->d.nx + 1);
  s->pg_buf_doubles = 3 * (size_t)world * s->d.batch * per; // three slots: step s lives in slot s mod 3
  const size_t bytes = s->pg_buf_doubles * sizeof(double) + 2 * ab2::kMaxPeers * sizeof(unsigned long long);
  CUDA_TRY(cudaMalloc(&s->pg_local, bytes));
  CUDA_TRY(cudaMemset(s->pg_local, 0, bytes));
  CUDA_TRY(cudaMalloc(&s->pg_done, sizeof(unsigned int)));
  CUDA_TRY(cudaMemset(s->pg_done, 0, sizeof(unsigned int)));
  s->pg_world = world;
  s->pg_rank = rank;
  cudaIpcMemHandle_t h;
  CUDA_TRY(cudaIpcGetMemHandle(&h, s->pg_local));
  static_assert(sizeof(h) == 64, "IPC handle size");
  std::memcpy(ipc_handle_out, &h, sizeof(h));
  return AB2_OK;
}

int ab2_gar_peer_gather_connect(ab2_gar_solver *s, const void *all_handles) {
  if (!s || !all_handles || !s->pg_local)
    return fail(AB2_ERR_STATE, "peer_gather_connect before peer_gather_init");
  CUDA_TRY(cudaSetDevice(s->d.device));
  for (int w = 0; w < s->pg_world; ++w) {
    void *base = s->pg_local;
    if (w != s->pg_rank) {
      cudaIpcMemHandle_t h;
      std::memcpy(&h, (const char *)all_handles + 64 * (size_t)w, sizeof(h));
      const cudaError_t e = cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) { // no peer access / IPC not permitted: leave the handle unconnected (callers fall back)
        cudaGetLastError();
        for (int v = 0; v < w; ++v) {
          if (v != s->pg_rank && s->pg_peer_base[v])
            cudaIpcCloseMemHandle(s->pg_peer_base[v]);
          s->pg_peer_base[v] = nullptr;
        }
        return fail(AB2_ERR_CUDA, std::string("peer_gather_connect: cudaIpcOpenMemHandle(rank ") + std::to_string(w) +
                                      "): " + cudaGetErrorString(e));
      }
    }
    s->pg_peer_base[w] = base;
    s->pg_ptrs.buf[w] = (double *)base;
    unsigned long long *fl = (unsigned long long *)((double *)base + s->pg_buf_doubles);
    s->pg_ptrs.data_flag[w] = fl;
    s->pg_ptrs.ack_flag[w] = fl + ab2::kMaxPeers;
  }
  return AB2_OK;
}

int ab2_gar_policy_allgather(ab2_gar_solver *s, void *stream) {
  if (!s || !s->pg_peer_base[0])
    return fail(AB2_ERR_STATE, "policy_allgather before peer_gather_connect");
  if (!s->have_backward)
    return fail(AB2_ERR_STATE, "policy_allgather before backward()");
  CUDA_TRY(cudaSetDevice(s->d.device));
  const long total = (long)s->d.batch * s->d.nu * (s->d.nx + 1);
  long blocks = (total + 255) / 256;
  if (blocks > s->p.num_sms * 2L)
    blocks = s->p.num_sms * 2L; // all resident at once: the last-CTA publication never waits on an unscheduled CTA
  s->pg_step += 1;
  if (s->pg_pushed_step == s->pg_step) // the sweep stored the blocks itself: publish the flags
    ab2::policy_publish_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(s->pg_ptrs, s->pg_world, s->pg_rank, s->pg_step);
  else
    ab2::policy_allgather_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(
        s->out[AB2_OUT_FB], s->out[AB2_OUT_FF], s->pg_ptrs, s->pg_world, s->pg_rank, s->d.batch, s->d.horizon, s->nr,
        s->d.nu, s->d.nx, s->pg_step, s->pg_done);
  CUDA_TRY(cudaGetLastError());
  s->launches += 1;
  return AB2_OK;
}

int ab2_gar_policy_allgather_wait(ab2_gar_solver *s, void *stream) {
  if (!s || !s->pg_peer_base[0] || s->pg_step == 0)
    return fail(AB2_ERR_STATE, "policy_allgather_wait before policy_allgather");
  CUDA_TRY(cudaSetDevice(s->d.device));
  static bool carve = false; // (an SM holds one shared-memory carve-out at a time: ask for the sweeps' so that this
  if (!carve) {              //  kernel can start while a sweep is resident)
    CUDA_TRY(cudaFuncSetAttribute(ab2::policy_wait_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                  (int)cudaSharedmemCarveoutMaxShared));
    carve = true;
  }
  ab2::policy_wait_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(s->pg_ptrs, s->pg_world, s->pg_rank, s->pg_step);
  CUDA_TRY(cudaGetLastError());
  s->launches += 1;
  return AB2_OK;
}

int ab2_gar_peer_gather_buffer(ab2_gar_solver *s, double **out, long *step) {
  if (!s || !out || !s->pg_local)
    return fail(AB2_ERR_STATE, "peer_gather_buffer before peer_gather_init");
  const size_t half = (size_t)(s->pg_step % 3) * s->pg_world * s->d.batch * s->d.nu * (s->d.nx + 1);
  *out = (double *)s->pg_local + half;
  if (step)
    *step = (long)s->pg_step;
  return AB2_OK;
}

int ab2_gar_pinned_alloc(size_t bytes, void **out) {
  if (!out)
    return fail(AB2_ERR_INVALID, "null argument");
  *out = nullptr;
  CUDA_TRY(cudaHostAlloc(out, bytes > 0 ? bytes : 1, cudaHostAllocPortable));
  return AB2_OK;
}
void ab2_gar_pinned_free(void *p) {
  if (p)
    cudaFreeHost(p);
}

long ab2_gar_launch_count(const ab2_gar_solver *s) { return s ? s->launches : 0; }

int ab2_gar_kernel_info(const ab2_gar_solver *s, int *group_lanes, int *smem_bytes_per_cta,
                        int *threads_per_cta, int *grid, int *regs_per_thread) {
  if (!s)
    return fail(AB2_ERR_INVALID, "null solver");
  int info[6] = {0, 0, 0, 0, 0, 0};
  CUDA_TRY(cudaSetDevice(s->d.device));
  if (s->k && s->variant != 9)
    CUDA_TRY(s->k->launch(s->p, s->variant, s->group_doubles, 0, info));
  else
    CUDA_TRY(ab2::launch_block(s->p, s->d.nx, s->d.nu, s->d.nc, 0, info));
  if (group_lanes)
    *group_lanes = info[0];
  if (smem_bytes_per_cta)
    *smem_bytes_per_cta = info[1];
  if (threads_per_cta)
    *threads_per_cta = info[2];
  if (grid)
    *grid = info[3];
  if (regs_per_thread)
    *regs_per_thread = info[4] | (info[5] << 16); /* high half: resident CTAs per SM */
  return AB2_OK;
}

} // extern "C"
