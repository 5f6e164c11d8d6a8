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
#include "kkt_error.h"
#include "linesearch.h"
#include "lq_adjoint.h"
#include "lq_resolve.h"
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
} // namespace

struct ab2_gar_solver {
  ab2_gar_dims d;
  const ab2::KernelEntry *k;
  int srec, trec, nr;
  ab2::SweepParams p;
  // owned device storage
  double *own_stage = nullptr, *own_term = nullptr, *own_G0 = nullptr, *own_g0 = nullptr;
  double *own_stage_sym = nullptr; // triangle-packed stage records as uploaded by ab2_gar_sweep_host_sym
  double *gains_tmp = nullptr, *kkt_tmp = nullptr, *theta_dev = nullptr, *ls_tmp = nullptr;
  double *fddp_slack = nullptr, *fddp_G0 = nullptr, *fddp_g0 = nullptr, *fddp_vx = nullptr;
  double *inner_tmp = nullptr; // [batch][2] per-instance scalars of multipliers / criterion, for host destinations
  double *mu_dev = nullptr;    // [batch] host-given per-instance mu of the *_v sweeps, staged for the kernels
  double *adj_stage = nullptr, *adj_term = nullptr, *adj_g0 = nullptr; // the adjoint problem of ab2_gar_adjoint
  double *tan_rho = nullptr; // rho of ab2_gar_tangent, in the solution's layouts (xs, us, vs, vsT, lam0, lams)
  double *ref_buf = nullptr;   // ab2_gar_refine's residual (rhs layout) and correction (out layout)
  double *ref_norms = nullptr; // staging of host norms of ab2_gar_refine / refine_many, ref_norms_n doubles
  size_t ref_norms_n = 0;
  int nth = 0; // parameter dimension of the value function outputs (= nx in leg mode)
  int rec_nth = 0; // parameter blocks carried by the knot records (0 in leg mode)
  int legs = 0;    // >= 2: gar::ParallelRiccatiSolver (leg mode)
  bool dense = false; // gar::RiccatiSolverDense (one CTA per instance, stage-dense KKT): FF/FB have nu+nc+2nx rows
  // O(1) cycleAppend: ring heads.  fac_head: physical slot of stage knot 0 in the per-knot FACTOR arrays
  // (FF, FB, VXX, VX) -- non-zero only between a cycle_append and the next backward, which rewrites every slot
  // in place; seen by the getters only.  p.stage_head: the same for the solver-owned copy of the stage records,
  // read by the kernels through stage_slot().
  int fac_head = 0;
  double *cond = nullptr;
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
  double *out[AB2_OUT_COUNT] = {};
  size_t out_doubles[AB2_OUT_COUNT] = {};
  size_t out_alloc[AB2_OUT_COUNT] = {}; // doubles allocated behind out[w] (>= out_doubles[w])
  size_t out_rec[AB2_OUT_COUNT] = {};  // doubles per knot (or per instance)
  int out_knots[AB2_OUT_COUNT] = {};   // knots per instance (1 for per-instance arrays)
  int *status = nullptr, *pivstat = nullptr;
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
  for (int w = 0; w < AB2_OUT_COUNT; ++w) {
    // (+2: the forward pass of the CTA-per-instance kernel fetches odd-sized gain records
    // with 16-byte granularity, up to one double past the end of the array)
    size_t n = s->out_doubles[w];
    if (w == AB2_OUT_VXX && s->k && vxx_packed_total > n)
      n = vxx_packed_total;
    const size_t bytes = (n > 0 ? n + 2 : 2) * sizeof(double);
    s->out_alloc[w] = bytes / sizeof(double);
    cudaError_t e = cudaMalloc(&s->out[w], bytes);
    if (e == cudaSuccess)
      e = cudaMemset(s->out[w], 0, bytes);
    if (e != cudaSuccess) {
      ab2_gar_destroy(s);
      return fail(AB2_ERR_CUDA, std::string("cudaMalloc outputs: ") + cudaGetErrorString(e));
    }
  }
  {
    cudaError_t e = cudaMalloc(&s->status, sizeof(int) * B);
    if (e == cudaSuccess)
      e = cudaMemset(s->status, 0, sizeof(int) * B);
    if (e != cudaSuccess) {
      ab2_gar_destroy(s);
      return fail(AB2_ERR_CUDA, std::string("cudaMalloc status: ") + cudaGetErrorString(e));
    }
  }
  {
    cudaError_t e = cudaMalloc(&s->pivstat, sizeof(int) * B);
    if (e == cudaSuccess)
      e = cudaMemset(s->pivstat, 0, sizeof(int) * B);
    if (e != cudaSuccess) {
      ab2_gar_destroy(s);
      return fail(AB2_ERR_CUDA, std::string("cudaMalloc pivstat: ") + cudaGetErrorString(e));
    }
  }
  if (legs > 1) {
    const size_t td = (size_t)d.nc0 + (size_t)d.nx * (2 * legs - 1);
    cudaError_t e = cudaMalloc(&s->cond, sizeof(double) * B * td);
    if (e == cudaSuccess)
      e = cudaMemset(s->cond, 0, sizeof(double) * B * td);
    if (e != cudaSuccess) {
      ab2_gar_destroy(s);
      return fail(AB2_ERR_CUDA, std::string("cudaMalloc cond: ") + cudaGetErrorString(e));
    }
  }
  ab2::SweepParams &p = s->p;
  std::memset(&p, 0, sizeof(p));
  p.legs = legs;
  p.cond = s->cond;
  p.N = N;
  p.nct = d.nct;
  p.nc0 = d.nc0;
  p.batch = B;
  p.ff = s->out[AB2_OUT_FF];
  p.fb = s->out[AB2_OUT_FB];
  p.Vxx = s->out[AB2_OUT_VXX];
  if (s->k)
    p.Vxx0 = p.Vxx + (size_t)B * (N + 1) * ab2::vxx_packed_doubles(nx);
  p.vx = s->out[AB2_OUT_VX];
  p.ffT = s->out[AB2_OUT_FFT];
  p.fbT = s->out[AB2_OUT_FBT];
  p.kkt0 = s->out[AB2_OUT_KKT0];
  p.xs = s->out[AB2_OUT_XS];
  p.us = s->out[AB2_OUT_US];
  p.vs = s->out[AB2_OUT_VS];
  p.vsT = s->out[AB2_OUT_VST];
  p.lbd0 = s->out[AB2_OUT_LBD0];
  p.lbdas = s->out[AB2_OUT_LBDAS];
  p.status = s->status;
  p.pivstat = s->pivstat;
  p.nth = nth;
  p.theta = nullptr;
  p.fth = s->out[AB2_OUT_FTH];
  p.Vxt = s->out[AB2_OUT_VXT];
  p.Vtt = s->out[AB2_OUT_VTT];
  p.vt = s->out[AB2_OUT_VT];
  p.kkt0fth = s->out[AB2_OUT_KKT0FTH];
  p.thGrad = s->out[AB2_OUT_THGRAD];
  p.thHess = s->out[AB2_OUT_THHESS];
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
  cudaSetDevice(s->d.device);
  for (int w = 0; w < AB2_OUT_COUNT; ++w)
    if (s->out[w])
      cudaFree(s->out[w]);
  if (s->status)
    cudaFree(s->status);
  if (s->pivstat)
    cudaFree(s->pivstat);
  for (int w = 0; w < s->pg_world; ++w)
    if (w != s->pg_rank && s->pg_peer_base[w])
      cudaIpcCloseMemHandle(s->pg_peer_base[w]);
  if (s->pg_local)
    cudaFree(s->pg_local);
  if (s->pg_done)
    cudaFree(s->pg_done);
  for (double *q : {s->own_stage_sym, s->own_stage, s->own_term, s->own_G0, s->own_g0, s->gains_tmp, s->kkt_tmp, s->theta_dev, s->cond, s->ls_tmp, s->fddp_slack, s->fddp_G0,
                    s->fddp_g0, s->fddp_vx, s->inner_tmp, s->mu_dev, s->adj_stage, s->adj_term, s->adj_g0, s->tan_rho,
                    s->ref_buf, s->ref_norms})
    if (q)
      cudaFree(q);
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
    auto up = [&](double *&own, const double *src, size_t n, const double *&dst) -> int {
      if (!src)
        return AB2_OK;
      if (!own)
        CUDA_TRY(cudaMalloc(&own, (n > 0 ? n : 1) * sizeof(double)));
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
  s->have_problem = s->p.stage && s->p.term && (s->p.G0 || s->d.nc0 == 0) && (s->p.g0 || s->d.nc0 == 0);
  if (s->d.horizon == 0 && s->p.term)
    s->have_problem = true;
  s->factor_current = false;
  s->epoch += 1;
  return AB2_OK;
}

// The configured backward runs the warp-per-instance kernel, which stores Vxx packed.
static bool warp_kernel(const ab2_gar_solver *s) { return s->k && s->variant != 9; }

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
  q.ff += b * s->out_knots[AB2_OUT_FF] * s->out_rec[AB2_OUT_FF];
  q.fb += b * s->out_knots[AB2_OUT_FB] * s->out_rec[AB2_OUT_FB];
  if (warp_kernel(s)) {
    q.Vxx += b * (N + 1) * ab2::vxx_packed_doubles(nx);
    q.Vxx0 += b * nx * nx;
  } else {
    q.Vxx += b * s->out_knots[AB2_OUT_VXX] * s->out_rec[AB2_OUT_VXX];
  }
  q.vx +=b * s->out_knots[AB2_OUT_VX] * s->out_rec[AB2_OUT_VX];
  q.ffT += b * s->out_rec[AB2_OUT_FFT];
  q.fbT += b * s->out_rec[AB2_OUT_FBT];
  q.kkt0 += b * s->out_rec[AB2_OUT_KKT0];
  q.xs += b * s->out_knots[AB2_OUT_XS] * s->out_rec[AB2_OUT_XS];
  q.us += b * s->out_knots[AB2_OUT_US] * s->out_rec[AB2_OUT_US];
  q.vs += b * s->out_knots[AB2_OUT_VS] * s->out_rec[AB2_OUT_VS];
  q.vsT += b * s->out_rec[AB2_OUT_VST];
  q.lbd0 += b * s->out_rec[AB2_OUT_LBD0];
  q.lbdas += b * s->out_knots[AB2_OUT_LBDAS] * s->out_rec[AB2_OUT_LBDAS];
  q.status += b;
  q.pivstat += b;
  if (s->nth > 0) {
    q.fth += b * s->out_knots[AB2_OUT_FTH] * s->out_rec[AB2_OUT_FTH];
    q.Vxt += b * s->out_knots[AB2_OUT_VXT] * s->out_rec[AB2_OUT_VXT];
    q.Vtt += b * s->out_knots[AB2_OUT_VTT] * s->out_rec[AB2_OUT_VTT];
    q.vt += b * s->out_knots[AB2_OUT_VT] * s->out_rec[AB2_OUT_VT];
    q.kkt0fth += b * s->out_rec[AB2_OUT_KKT0FTH];
    q.thGrad += b * s->out_rec[AB2_OUT_THGRAD];
    q.thHess += b * s->out_rec[AB2_OUT_THHESS];
    if (q.theta)
      q.theta += b * s->nth;
  }
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
  if (!mueq_b)
    s->p.mueq = mueq;
  s->p.do_bwd = bwd;
  s->p.do_fwd = fwd;
  ab2::SweepParams q = s->p;
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
  if (bwd) {
    s->have_backward = true;
    s->fac_head = 0; // every factor slot was rewritten in knot order
    s->vxx_packed = warp_kernel(s);
    s->factor_current = true;
    s->epoch += 1;
    s->primal_factor = true;
  }
  s->have_forward = fwd != 0; // a backward-only launch invalidates the previous trajectory
  s->have_primal = fwd != 0 && s->primal_factor;
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
  if (!s->mu_dev)
    CUDA_TRY(cudaMalloc(&s->mu_dev, (size_t)s->d.batch * sizeof(double)));
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
      if (!s->theta_dev)
        CUDA_TRY(cudaMalloc(&s->theta_dev, (size_t)s->d.batch * s->nth * sizeof(double)));
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
// fields in the solution's layouts, `blocks` instances (batch, or nrhs * batch)
static Fields sol_fields(const ab2_gar_solver *s, const char *what, const double *const p[6], size_t blocks) {
  const ab2_gar_dims &d = s->d;
  const int N = d.horizon;
  const size_t per[6] = {(size_t)(N + 1) * d.nx, (size_t)N * d.nu, (size_t)N * d.nc, (size_t)d.nct, (size_t)d.nc0,
                         (size_t)N * d.nx};
  Fields f{what, kSolNames, {}, {}, 6};
  for (int i = 0; i < 6; ++i) {
    f.p[i] = p[i];
    f.n[i] = blocks * per[i];
  }
  return f;
}
// fields in the problem's record layouts (stage, term, G0, g0), `blocks` instances
static Fields rec_fields(const ab2_gar_solver *s, const char *what, const double *const p[4], size_t blocks) {
  const ab2_gar_dims &d = s->d;
  const size_t per[4] = {(size_t)d.horizon * s->srec, (size_t)s->trec, (size_t)d.nc0 * d.nx, (size_t)d.nc0};
  Fields f{what, kRecNames, {}, {}, 4};
  for (int i = 0; i < 4; ++i) {
    f.p[i] = p[i];
    f.n[i] = blocks * per[i];
  }
  return f;
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
// fields in resolve's rhs layouts (the same sizes as the solution's), `blocks` instances
static Fields rhs_fields(const ab2_gar_solver *s, const char *what, const double *const p[6], size_t blocks) {
  Fields f = sol_fields(s, what, p, blocks);
  f.names = kRhsNames;
  return f;
}
static const char *const kFacNames[6] = {"ff", "fb", "vxx", "vx", "fft", "fbt"};
// fields in ab2_gar_get's layouts of the factorisation (FF .. FBT, vxx as full blocks), `blocks` instances
static Fields fac_fields(const ab2_gar_solver *s, const char *what, const double *const p[6], size_t blocks) {
  const ab2_gar_dims &d = s->d;
  const size_t N = d.horizon, nx = d.nx, nr = d.nu + d.nc + d.nx;
  const size_t per[6] = {N * nr, N * nr * nx, (N + 1) * nx * nx, (N + 1) * nx, (size_t)d.nct, (size_t)d.nct * nx};
  Fields f{what, kFacNames, {}, {}, 6};
  for (int i = 0; i < 6; ++i) {
    f.p[i] = p[i];
    f.n[i] = blocks * per[i];
  }
  return f;
}
static const char *const kOutNames[AB2_OUT_COUNT] = {"FF",   "FB",    "VXX",  "VX",  "FFT",     "FBT",    "KKT0",
                                                     "XS",   "US",    "VS",   "VST", "LBD0",    "LBDAS",  "FTH",
                                                     "VXT",  "VTT",   "VT",   "KKT0FTH", "THGRAD", "THHESS"};
// the handle's own output arrays, as allocated
static Fields out_fields(const ab2_gar_solver *s) {
  Fields f{"the handle's output", kOutNames, {}, {}, AB2_OUT_COUNT};
  for (int w = 0; w < AB2_OUT_COUNT; ++w) {
    f.p[w] = s->out[w];
    f.n[w] = s->out_alloc[w];
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
  const ab2_gar_dims &d = s->d;
  const int B = d.batch, N = d.horizon, nx = d.nx;
  auto own = [&](double *&buf, size_t n) -> int {
    if (!buf)
      CUDA_TRY(cudaMalloc(&buf, (n > 0 ? n : 1) * sizeof(double)));
    return AB2_OK;
  };
  int rc;
  if ((rc = own(s->adj_stage, stage_total(s))) != AB2_OK || (rc = own(s->adj_term, (size_t)B * s->trec)) != AB2_OK ||
      (rc = own(s->adj_g0, (size_t)B * d.nc0)) != AB2_OK)
    return rc;
  const ab2::AdjointDims ad{B, N, nx, d.nu, d.nc, d.nct, d.nc0, s->srec, s->trec};
  // 1. the problem: same matrices, vectors = -cot (copy: cot)
  ab2::AdjointRecordArgs ra{ad, s->p.stage_head, s->p.stage, s->p.term, cot->xs, cot->us, cot->vs, cot->vsT,
                            cot->lam0, cot->lams, s->adj_stage, s->adj_term, s->adj_g0, copy};
  CUDA_TRY(ab2::launch_adjoint_records(ra, st));
  s->launches += 1;
  // 2. backward + forward on it; the problem pointers change in this launch's copy of the parameters only, and a
  //    sharded handle never publishes these gains to its peers
  if (!mu_dev)
    s->p.mueq = mueq;
  ab2::SweepParams q = s->p;
  q.stage = s->adj_stage;
  q.stage_head = 0;
  q.term = s->adj_term;
  q.g0 = s->adj_g0;
  q.mueq_b = mu_dev;
  q.peer_world = 0;
  if ((rc = run_kernels(s, q, 1, 1, st)) != AB2_OK)
    return rc;
  s->have_backward = true;
  s->have_forward = true;
  s->primal_factor = false; // the trajectory outputs are w or zdot, not the primal solution
  s->have_primal = false;
  s->fac_head = 0;
  s->vxx_packed = warp_kernel(s);
  s->factor_current = true;
  s->epoch += 1;
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
  const double *pp[6] = {primal->xs, primal->us, primal->vs, primal->vsT, primal->lam0, primal->lams};
  const Fields P = sol_fields(s, "primal", pp, s->d.batch);
  if (int rc = require(P, who))
    return rc;
  if (int rc = refuse_overlap(P, out_fields(s), who))
    return rc;
  if (int rc = check_mu(s, mueq, mueq_arr, who))
    return rc;
  const ab2_gar_dims &d = s->d;
  const int B = d.batch, N = d.horizon, nx = d.nx;
  cudaStream_t st;
  const double *mu_dev;
  if (int rc = begin_launch(s, mueq_arr, memspace, stream, &st, &mu_dev))
    return rc;
  // 1. + 2. the adjoint problem (vectors = -cotangent) and its solve
  int rc;
  if ((rc = solve_cotangent_problem(s, mueq, mu_dev, cot, false, st)) != AB2_OK)
    return rc;
  const ab2::AdjointDims ad{B, N, nx, d.nu, d.nc, d.nct, d.nc0, s->srec, s->trec};
  // 3. gradient records from the primal z and the adjoint w (the trajectory outputs): dh = -w, dK = -w z^T
  ab2::JacobianGradArgs ga{ad, 1,
                           primal->xs, primal->us, primal->vs, primal->vsT, primal->lam0, primal->lams,
                           s->out[AB2_OUT_XS], s->out[AB2_OUT_US], s->out[AB2_OUT_VS], s->out[AB2_OUT_VST],
                           s->out[AB2_OUT_LBD0], s->out[AB2_OUT_LBDAS],
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
  const double *pp[6] = {primal->xs, primal->us, primal->vs, primal->vsT, primal->lam0, primal->lams};
  if (int rc = require(sol_fields(s, "primal", pp, s->d.batch), who))
    return rc;
  if (int rc = check_mu(s, mueq, mueq_arr, who))
    return rc;
  const ab2_gar_dims &d = s->d;
  const int B = d.batch, N = d.horizon, nx = d.nx;
  cudaStream_t st;
  const double *mu_dev;
  if (int rc = begin_launch(s, mueq_arr, memspace, stream, &st, &mu_dev))
    return rc;
  const size_t nxs = (size_t)B * (N + 1) * nx, nus = (size_t)B * N * d.nu, nvs = (size_t)B * N * d.nc,
               nvT = (size_t)B * d.nct, nl0 = (size_t)B * d.nc0, nls = (size_t)B * N * nx;
  if (!s->tan_rho)
    CUDA_TRY(cudaMalloc(&s->tan_rho, (nxs + nus + nvs + nvT + nl0 + nls + 1) * sizeof(double)));
  double *rxs = s->tan_rho, *rus = rxs + nxs, *rvs = rus + nus, *rvT = rvs + nvs, *rl0 = rvT + nvT, *rls = rl0 + nl0;
  // 1. rho = Kdot z + hdot, in the solution's layouts
  const ab2::AdjointDims ad{B, N, nx, d.nu, d.nc, d.nct, d.nc0, s->srec, s->trec};
  ab2::JacobianRhsArgs ra{ad, 1, dot->stage, dot->term, dot->G0, dot->g0,
                          primal->xs, primal->us, primal->vs, primal->vsT, primal->lam0, primal->lams,
                          rxs, rus, rvs, rvT, rl0, rls};
  CUDA_TRY(ab2::launch_jacobian_rhs(ra, st));
  s->launches += 1;
  // 2. + 3. the tangent problem (vectors = rho) and its solve: the trajectory outputs become zdot
  const ab2_ls_iterate rho{rxs, rus, rvs, rvT, rl0, rls};
  return solve_cotangent_problem(s, mueq, mu_dev, &rho, true, st);
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
  const double *po[6] = {out->xs, out->us, out->vs, out->vsT, out->lam0, out->lams};
  const double *ph[6] = {rhs->q, rhs->r, rhs->d, rhs->dN, rhs->g0, rhs->f};
  if (int rc = require(sol_fields(s, "out", po, 1), who)) // (refused even at nrhs = 0)
    return rc;
  if (int rc = check_mu(s, mueq, mueq_arr, who))
    return rc;
  // the backward pass parks its per-knot vectors in the out arrays before it has read every rhs entry: an out array
  // that overlaps an rhs array would be read after it was overwritten
  if (int rc = refuse_overlap(rhs_fields(s, "rhs", ph, R), sol_fields(s, "out", po, R), who))
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
  const double *pc[6] = {cot->ff, cot->fb, cot->vxx, cot->vx, cot->fft, cot->fbt};
  const double *pg[4] = {grad->stage, grad->term, grad->G0, grad->g0};
  const Fields G = rec_fields(s, "grad", pg, d.batch);
  if (int rc = refuse_overlap(G, fac_fields(s, "cotangent", pc, d.batch), who))
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
  const double *po[6] = {out->ff, out->fb, out->vxx, out->vx, out->fft, out->fbt};
  const double *pd[4] = {dot->stage, dot->term, dot->G0, dot->g0};
  const Fields O = fac_fields(s, "out", po, d.batch);
  if (int rc = refuse_overlap(O, rec_fields(s, "tangent", pd, d.batch), who))
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
  const double *pp[6] = {primal->xs, primal->us, primal->vs, primal->vsT, primal->lam0, primal->lams};
  const double *pc[6] = {cot->xs, cot->us, cot->vs, cot->vsT, cot->lam0, cot->lams};
  const double *pw[6] = {work->xs, work->us, work->vs, work->vsT, work->lam0, work->lams};
  const double *pg[4] = {grad->stage, grad->term, grad->G0, grad->g0};
  const Fields P = sol_fields(s, "primal", pp, B), Z = sol_fields(s, "cotangent", pc, R),
               W = sol_fields(s, "work", pw, R), G = rec_fields(s, "grad", pg, R);
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
  const ab2::AdjointDims ad{d.batch, d.horizon, d.nx, d.nu, d.nc, d.nct, d.nc0, s->srec, s->trec};
  ab2::JacobianGradArgs ga{ad, nrhs,
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
  const double *pp[6] = {primal->xs, primal->us, primal->vs, primal->vsT, primal->lam0, primal->lams};
  const double *pd[4] = {dot->stage, dot->term, dot->G0, dot->g0};
  const double *pw[6] = {work->xs, work->us, work->vs, work->vsT, work->lam0, work->lams};
  const double *po[6] = {out->xs, out->us, out->vs, out->vsT, out->lam0, out->lams};
  const Fields P = sol_fields(s, "primal", pp, B), D = rec_fields(s, "dot", pd, R),
               W = sol_fields(s, "work", pw, R), O = sol_fields(s, "out", po, R);
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
  const ab2::AdjointDims ad{d.batch, d.horizon, d.nx, d.nu, d.nc, d.nct, d.nc0, s->srec, s->trec};
  ab2::JacobianRhsArgs ra{ad, nrhs, dot->stage, dot->term, dot->G0, dot->g0,
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
  double *ndev = nullptr;
  if (norms) {
    if (device_accessible(norms)) {
      ndev = norms;
    } else {
      if (s->ref_norms_n < nnorm) {
        if (s->ref_norms)
          CUDA_TRY(cudaFree(s->ref_norms));
        s->ref_norms = nullptr;
        s->ref_norms_n = 0;
        CUDA_TRY(cudaMalloc(&s->ref_norms, nnorm * sizeof(double)));
        s->ref_norms_n = nnorm;
      }
      ndev = s->ref_norms;
    }
    CUDA_TRY(cudaMemsetAsync(ndev, 0, nnorm * sizeof(double), st)); // the maxima meet by atomicMax from 0
  }
  const ab2::AdjointDims ad{B, N, d.nx, d.nu, d.nc, d.nct, d.nc0, s->srec, s->trec};
  auto residual = [&](int col, bool write) -> int {
    ab2::RefineResidualArgs a{};
    a.d = ad;
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
    a.norms = ndev;
    a.nstride = steps + 1;
    a.col = col;
    CUDA_TRY(ab2::launch_refine_residual(a, st));
    s->launches += 1;
    return AB2_OK;
  };
  const size_t no[6] = {R * (N + 1) * d.nx, R * N * d.nu, R * N * d.nc, R * d.nct, R * d.nc0, R * N * d.nx};
  const ab2_lq_rhs rr{r->xs, r->us, r->vs, r->vsT, r->lam0, r->lams};
  for (int k = 0; k < steps; ++k) {
    if (int rc = residual(k, true)) // r = K z + h
      return rc;
    if (int rc = run_resolve(s, mueq, mu_dev, nrhs, &rr, dz, st)) // dz = -K^-1 r
      return rc;
    ab2::RefineUpdateArgs u{{z->xs, z->us, z->vs, z->vsT, z->lam0, z->lams},
                            {dz->xs, dz->us, dz->vs, dz->vsT, dz->lam0, dz->lams},
                            {(long)no[0], (long)no[1], (long)no[2], (long)no[3], (long)no[4], (long)no[5]}};
    CUDA_TRY(ab2::launch_refine_update(u, st)); // z += dz
    s->launches += 1;
  }
  if (ndev) {
    if (int rc = residual(steps, false)) // the last column: the norm of the refined iterate
      return rc;
    if (ndev != norms)
      CUDA_TRY(cudaMemcpyAsync(norms, ndev, nnorm * sizeof(double), cudaMemcpyDeviceToHost, st));
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
  const ab2_gar_dims &d = s->d;
  const int B = d.batch, N = d.horizon, nx = d.nx;
  cudaStream_t st;
  const double *mu_dev;
  if (int rc = begin_launch(s, mueq_arr, memspace, stream, &st, &mu_dev))
    return rc;
  const size_t nxs = (size_t)B * (N + 1) * nx, nus = (size_t)B * N * d.nu, nvs = (size_t)B * N * d.nc,
               nvT = (size_t)B * d.nct, nl0 = (size_t)B * d.nc0, nls = (size_t)B * N * nx,
               one = nxs + nus + nvs + nvT + nl0 + nls;
  if (!s->ref_buf)
    CUDA_TRY(cudaMalloc(&s->ref_buf, (2 * one + 1) * sizeof(double)));
  auto split = [&](double *p) {
    ab2_ls_trial t;
    t.xs = p;
    t.us = t.xs + nxs;
    t.vs = t.us + nus;
    t.vsT = t.vs + nvs;
    t.lam0 = t.vsT + nvT;
    t.lams = t.lam0 + nl0;
    return t;
  };
  const ab2_ls_trial r = split(s->ref_buf), dz = split(s->ref_buf + one);
  const ab2_ls_trial z{s->out[AB2_OUT_XS], s->out[AB2_OUT_US], s->out[AB2_OUT_VS], s->out[AB2_OUT_VST],
                       s->out[AB2_OUT_LBD0], s->out[AB2_OUT_LBDAS]};
  return run_refine(s, mueq, mu_dev, 1, steps, true, nullptr, &z, &r, &dz, norms, st);
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
  const double *ph[6] = {rhs->q, rhs->r, rhs->d, rhs->dN, rhs->g0, rhs->f};
  const double *pz[6] = {z->xs, z->us, z->vs, z->vsT, z->lam0, z->lams};
  const double *pr[6] = {work->q, work->r, work->d, work->dN, work->g0, work->f};
  const double *pd[6] = {work->xs, work->us, work->vs, work->vsT, work->lam0, work->lams};
  const Fields H = rhs_fields(s, "rhs", ph, R), Z = sol_fields(s, "z", pz, R), WR = rhs_fields(s, "work", pr, R),
               WD = sol_fields(s, "work", pd, R);
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
  auto own = [&](double *&buf, size_t n) -> int {
    if (!buf)
      CUDA_TRY(cudaMalloc(&buf, (n > 0 ? n : 1) * sizeof(double)));
    return AB2_OK;
  };
  int rc;
  if ((rc = own(s->own_stage, stage_total(s))) != AB2_OK || (rc = own(s->own_term, (size_t)d.batch * s->trec)) != AB2_OK ||
      (rc = own(s->own_G0, (size_t)d.batch * d.nc0 * d.nx)) != AB2_OK || (rc = own(s->own_g0, (size_t)d.batch * d.nc0)) != AB2_OK)
    return rc;
  CUDA_TRY(ab2::launch_lq_assemble(*in, preg_b, mu_inv_b, s->own_stage, s->own_term, s->own_G0, s->own_g0, d.batch, d.horizon, d.nx,
                                   d.nu, d.nc, d.nct, d.nc0, s->srec, s->trec, (cudaStream_t)stream));
  s->launches += d.horizon > 0 ? 2 : 1;
  s->p.stage = s->own_stage;
  s->p.stage_head = 0;
  s->p.term = s->own_term;
  s->p.G0 = s->own_G0;
  s->p.g0 = s->own_g0;
  s->have_problem = true;
  s->factor_current = false;
  s->epoch += 1;
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
  long blocks = (long)((n + 255) / 256);
  if (blocks > s->p.num_sms * 8L)
    blocks = s->p.num_sms * 8L;
  ab2::vxx_expand_kernel<<<(int)blocks, 256, 0, st>>>(s->out[AB2_OUT_VXX], s->p.Vxx0, out, s->d.horizon, s->d.nx, head,
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
                     s->d.horizon, dst, memspace == AB2_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                     (cudaStream_t)stream);
  if (n[what])
    CUDA_TRY(cudaMemcpyAsync(dst, ptrs[what], n[what] * sizeof(double),
                             memspace == AB2_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                             (cudaStream_t)stream));
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
  auto own = [&](double *&buf, size_t n) -> int {
    if (!buf)
      CUDA_TRY(cudaMalloc(&buf, (n > 0 ? n : 1) * sizeof(double)));
    return AB2_OK;
  };
  int rc;
  if ((rc = own(s->own_stage, stage_total(s))) != AB2_OK || (rc = own(s->own_term, (size_t)B * s->trec)) != AB2_OK ||
      (rc = own(s->own_G0, (size_t)B * nc0 * nx)) != AB2_OK || (rc = own(s->own_g0, (size_t)B * nc0)) != AB2_OK)
    return rc;
  const size_t srec_sym = ab2_gar_stage_record_doubles_sym(nx, s->d.nu, s->d.nc);
  if (sym && (rc = own(s->own_stage_sym, (size_t)B * N * srec_sym)) != AB2_OK)
    return rc;
  s->p.stage = s->own_stage;
  s->p.stage_head = 0;
  s->p.term = s->own_term;
  s->p.G0 = s->own_G0;
  s->p.g0 = s->own_g0;
  s->have_problem = true;
  if (!mueq_b)
    s->p.mueq = mueq;
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
        long blocks = (nrec * (long)s->srec + 255) / 256;
        if (blocks > s->p.num_sms * 8L)
          blocks = s->p.num_sms * 8L;
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
        ab2::expand_sym_kernel<<<(int)blocks, 256, s->srec * sizeof(int), st>>>(
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
  s->have_backward = true;
  s->have_forward = true;
  s->primal_factor = true;
  s->have_primal = true;
  s->fac_head = 0;
  s->vxx_packed = warp_kernel(s);
  s->factor_current = true;
  s->epoch += 1;
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
                     s->out_knots[what], dst, memspace == AB2_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                     (cudaStream_t)stream);
  CUDA_TRY(cudaMemcpyAsync(dst, s->out[what], s->out_doubles[what] * sizeof(double),
                           memspace == AB2_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
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
    return copy_ring(s->out[what], rec, knots, s->d.horizon, s->fac_head, b0, nb, t0, nt, dst,
                     memspace == AB2_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, (cudaStream_t)stream);
  const double *src = s->out[what] + ((size_t)b0 * knots + t0) * rec;
  CUDA_TRY(cudaMemcpy2DAsync(dst, (size_t)nt * rec * sizeof(double), src, (size_t)knots * rec * sizeof(double),
                             (size_t)nt * rec * sizeof(double), (size_t)nb,
                             memspace == AB2_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                             (cudaStream_t)stream));
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
  const long total = (long)s->d.batch * s->d.nu * (s->d.nx + 1);
  const int threads = 256;
  long blocks = (total + threads - 1) / threads;
  if (blocks > s->p.num_sms * 8L)
    blocks = s->p.num_sms * 8L;
  ab2::first_step_policy_kernel<<<(int)blocks, threads, 0, (cudaStream_t)stream>>>(
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
  double *out = dst;
  if (memspace != AB2_DEVICE) { // stage on the device, then one copy
    if (!s->gains_tmp)
      CUDA_TRY(cudaMalloc(&s->gains_tmp, total * sizeof(double)));
    out = s->gains_tmp;
  }
  long blocks = ((long)total + 255) / 256;
  if (blocks > s->p.num_sms * 8L)
    blocks = s->p.num_sms * 8L;
  ab2::gains_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(s->out[AB2_OUT_FB], s->out[AB2_OUT_FF], out, nrec,
                                                                    s->nr, s->d.nx, s->d.horizon, s->fac_head);
  CUDA_TRY(cudaGetLastError());
  s->launches += 1;
  if (memspace != AB2_DEVICE)
    CUDA_TRY(cudaMemcpyAsync(dst, out, total * sizeof(double), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return AB2_OK;
}

static int kkt_error_impl(ab2_gar_solver *s, double mueq, const double *mueq_b, double *dst, int memspace, void *stream) {
  if (!s || !dst)
    return fail(AB2_ERR_INVALID, "bad argument");
  if (!s->have_problem || !s->have_backward || !s->have_forward)
    return fail(AB2_ERR_STATE, "kkt_error needs a problem and a completed sweep (no forward pass since the last backward)");
  if (s->rec_nth > 0)
    return fail(AB2_ERR_UNSUPPORTED, "kkt_error: parametric problems (nth > 0) are not supported");
  CUDA_TRY(cudaSetDevice(s->d.device));
  if (!s->kkt_tmp)
    CUDA_TRY(cudaMalloc(&s->kkt_tmp, (size_t)s->d.batch * 3 * sizeof(double)));
  ab2::KktErrorArgs a;
  a.batch = s->d.batch;
  a.N = s->d.horizon;
  a.nx = s->d.nx;
  a.nu = s->d.nu;
  a.nc = s->d.nc;
  a.nct = s->d.nct;
  a.nc0 = s->d.nc0;
  a.srec = s->srec;
  a.trec = s->trec;
  a.stage_head = s->p.stage_head;
  a.mueq = mueq;
  a.mueq_b = mueq_b;
  a.stage = s->p.stage;
  a.term = s->p.term;
  a.G0 = s->p.G0;
  a.g0 = s->p.g0;
  a.xs = s->out[AB2_OUT_XS];
  a.us = s->out[AB2_OUT_US];
  a.vs = s->out[AB2_OUT_VS];
  a.vsT = s->out[AB2_OUT_VST];
  a.lbd0 = s->out[AB2_OUT_LBD0];
  a.lbdas = s->out[AB2_OUT_LBDAS];
  a.out = (memspace == AB2_DEVICE) ? dst : s->kkt_tmp;
  CUDA_TRY(ab2::launch_kkt_error(a, (cudaStream_t)stream));
  s->launches += 1;
  if (memspace != AB2_DEVICE)
    CUDA_TRY(cudaMemcpyAsync(dst, s->kkt_tmp, (size_t)s->d.batch * 3 * sizeof(double), cudaMemcpyDeviceToHost,
                             (cudaStream_t)stream));
  return AB2_OK;
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
  CUDA_TRY(cudaMemcpyAsync(dst, s->status, sizeof(int) * s->d.batch,
                           memspace == AB2_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                           (cudaStream_t)stream));
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
  a.dxs = s->out[AB2_OUT_XS];
  a.dus = s->out[AB2_OUT_US];
  a.dvs = s->out[AB2_OUT_VS];
  a.dvsT = s->out[AB2_OUT_VST];
  a.dlam0 = s->out[AB2_OUT_LBD0];
  a.dlams = s->out[AB2_OUT_LBDAS];
  return a;
}
static int ls_result(ab2_gar_solver *s, double *dst, int memspace, cudaStream_t st, double **dev) {
  if (memspace == AB2_DEVICE) {
    *dev = dst;
    return AB2_OK;
  }
  if (!s->ls_tmp)
    CUDA_TRY(cudaMalloc(&s->ls_tmp, (size_t)s->d.batch * sizeof(double)));
  *dev = s->ls_tmp;
  (void)st;
  return AB2_OK;
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
  double *dev = nullptr;
  if (int rc = ls_result(s, dst, memspace, (cudaStream_t)stream, &dev))
    return rc;
  CUDA_TRY(ab2::launch_directional_derivative(ls_args(s), Lxs, Lus, dev, (cudaStream_t)stream));
  s->launches += 1;
  if (memspace != AB2_DEVICE)
    CUDA_TRY(cudaMemcpyAsync(dst, dev, (size_t)s->d.batch * sizeof(double), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return AB2_OK;
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
  double *dev = nullptr;
  if (int rc = ls_result(s, dst, memspace, (cudaStream_t)stream, &dev))
    return rc;
  CUDA_TRY(ab2::launch_al_value(d.batch, d.horizon, d.nx, d.nc, d.nct, d.nc0, plus->lam0, plus->lams, plus->vs, plus->vsT,
                                cost, mudyn, mucstr, mudyn_b, mucstr_b, dev, (cudaStream_t)stream));
  s->launches += 1;
  if (memspace != AB2_DEVICE)
    CUDA_TRY(cudaMemcpyAsync(dst, dev, (size_t)d.batch * sizeof(double), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return AB2_OK;
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
// device destination of a [batch][2] result: the caller's buffer or the handle's scratch (copied out afterwards)
static int inner_result(ab2_gar_solver *s, double *dst, int memspace, double **dev) {
  if (memspace == AB2_DEVICE) {
    *dev = dst;
    return AB2_OK;
  }
  if (!s->inner_tmp)
    CUDA_TRY(cudaMalloc(&s->inner_tmp, (size_t)s->d.batch * 2 * sizeof(double)));
  *dev = s->inner_tmp;
  return AB2_OK;
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
  double *dev = nullptr;
  if (int rc = inner_result(s, dst, memspace, &dev))
    return rc;
  CUDA_TRY(ab2::launch_multipliers(inner_dims(s), *in, mu_b, mu_dyn_b, *out, dev, (cudaStream_t)stream));
  s->launches += 1;
  if (memspace != AB2_DEVICE)
    CUDA_TRY(cudaMemcpyAsync(dst, dev, (size_t)d.batch * 2 * sizeof(double), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return AB2_OK;
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
  double *dev = nullptr;
  if (int rc = inner_result(s, dst, memspace, &dev))
    return rc;
  CUDA_TRY(ab2::launch_criterion(inner_dims(s), Lxs, Lus, init_value, slack, Lv, Lv_N, dev, (cudaStream_t)stream));
  s->launches += 1;
  if (memspace != AB2_DEVICE)
    CUDA_TRY(cudaMemcpyAsync(dst, dev, (size_t)d.batch * 2 * sizeof(double), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return AB2_OK;
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
  auto own = [&](double *&buf, size_t n) -> int {
    if (!buf)
      CUDA_TRY(cudaMalloc(&buf, (n > 0 ? n : 1) * sizeof(double)));
    return AB2_OK;
  };
  int rc;
  if ((rc = own(s->fddp_slack, (size_t)B * N * nx)) != AB2_OK || (rc = own(s->fddp_G0, (size_t)B * nx * nx)) != AB2_OK ||
      (rc = own(s->fddp_g0, (size_t)B * nx)) != AB2_OK || (rc = own(s->fddp_vx, (size_t)B * (N + 1) * nx)) != AB2_OK)
    return rc;
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
  if ((rc = assemble_impl(s, &lq, preg_b, nullptr, stream)) != AB2_OK)
    return rc;
  if ((rc = ab2_gar_backward(s, 1.0, stream)) != AB2_OK) // (mueq is unused without constraints)
    return rc;
  double *vxo = Vx_out ? Vx_out : s->fddp_vx;
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
  CUDA_TRY(cudaMemcpyAsync(dst, s->pivstat, sizeof(int) * s->d.batch,
                           memspace == AB2_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                           (cudaStream_t)stream));
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
    s->fac_head = (s->fac_head + 1) % N;
    const int slot = (N - 1 + s->fac_head) % N; // physical slot of the new stage knot N-1 (= the old knot 0's)
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
  s->have_backward = false;
  s->have_forward = false;
  s->have_primal = false;
  s->factor_current = false;
  s->epoch += 1;
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
