// block_kernel.cu -- device context, kernel and launcher of the CTA-per-instance sweep
// for run-time dimensions (riccati_block.cuh).  One CTA walks the whole horizon of one
// instance; the stage records stream in by TMA bulk copies (two mbarrier-tracked parts),
// the forward gains through a ring of up to 8 TMA-filled slots.
#include <cuda_runtime.h>

#include "riccati_block.cuh"
#include "riccati_dense.cuh"
#include "riccati_block_launch.h"
#include "riccati_launch.cuh"

namespace ab2 {

struct BlockDevCtx {
  int tid, nthreads, warp, lane, nwarps;
  uint32_t bar0;  // shared address of the CTA's NBAR mbarriers
  uint32_t phase; // bit p = parity to wait for on barrier p

  __device__ __forceinline__ void sync() { __syncthreads(); }
  // CTA barrier that also ORs a flag over all threads
  __device__ __forceinline__ int sync_or(int v) { return __syncthreads_or(v); }
  // barrier over the first `nth` threads (whole warps) of the CTA: named barrier 1
  __device__ __forceinline__ void sync_sub(int nth) { asm volatile("bar.sync 1, %0;" ::"r"(nth) : "memory"); }
  __device__ __forceinline__ void wsync() { __syncwarp(); }
  __device__ __forceinline__ void atomic_or(int *q, int v) { atomicOr(q, v); }
  __device__ __forceinline__ void atomic_add(int *q, int v) { atomicAdd(q, v); }
  // generic-proxy writes of this thread (shared and global) ordered before later TMA accesses
  __device__ __forceinline__ void proxy_fence() { asm volatile("fence.proxy.async;" ::: "memory"); }
  __device__ __forceinline__ double shfl(double v, int src) { return __shfl_sync(0xffffffffu, v, src); }
  __device__ __forceinline__ bool all(bool p) { return __all_sync(0xffffffffu, p); }
  __device__ __forceinline__ void mma(double (&d)[2], double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(d[0]), "+d"(d[1])
                 : "d"(a), "d"(b));
  }
  __device__ __forceinline__ void init(uint64_t *bars) {
    bar0 = smem_u32(bars);
    phase = 0;
    if (tid == 0) {
      for (int b = 0; b < NBAR; ++b)
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar0 + 8 * b));
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
  }
  // `nd` doubles (even, 16-byte aligned both sides) global -> shared; called by every
  // thread after a CTA barrier that orders the last generic-proxy accesses to dst.
  __device__ __forceinline__ void issue_copy(int part, double *dst, const double *src, int nd) {
    if (tid == 0) {
      const uint32_t bar = bar0 + 8 * part;
      const uint32_t bytes = (uint32_t)nd * 8u;
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
      const uint32_t CH = 32768u;
      for (uint32_t o = 0; o < bytes; o += CH) {
        const uint32_t n = bytes - o < CH ? bytes - o : CH;
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                smem_u32(dst) + o),
            "l"(reinterpret_cast<const char *>(src) + o), "r"(n), "r"(bar)
            : "memory");
      }
    }
  }
  __device__ __forceinline__ void wait_copy(int part) {
    const uint32_t bar = bar0 + 8 * part;
    uint32_t done = 0;
    while (!done) {
      asm volatile("{\n\t.reg .pred p;\n\t"
                   "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                   "selp.u32 %0, 1, 0, p;\n\t}"
                   : "=r"(done)
                   : "r"(bar), "r"((phase >> part) & 1u)
                   : "memory");
    }
    phase ^= (1u << part);
  }
};

// MAXREG 128: two or more CTAs per SM for the shapes whose buffers allow it; 255: the
// large shapes, which own the SM anyway.
// PI: per-instance mu (SweepParams::mueq_b, the *_v launches); false = the scalar p.mueq
template <int MAXREG, class D, bool PI>
__global__ void __launch_bounds__(256) __maxnreg__(MAXREG)
    riccati_block_kernel(const SweepParams p, const D d) {
  extern __shared__ __align__(16) double smem[];
  BlockDevCtx ctx;
  ctx.tid = threadIdx.x;
  ctx.nthreads = blockDim.x;
  ctx.warp = threadIdx.x >> 5;
  ctx.lane = threadIdx.x & 31;
  ctx.nwarps = blockDim.x >> 5;
  ctx.init(reinterpret_cast<uint64_t *>(smem + d.s_end));
  const int legs = p.legs > 1 ? p.legs : 1; // leg mode: a work item is one (instance, leg)
  for (int item = blockIdx.x; item < p.batch * legs; item += gridDim.x) {
    if constexpr (PI) {
      riccati_block_sweep(ctx, p, d, item / legs, smem, item % legs, InstanceMu());
      flag_bad_mu(p, item / legs, d.nc > 0 || p.nct > 0, ctx.tid == 0);
    } else {
      riccati_block_sweep(ctx, p, d, item / legs, smem, item % legs);
    }
    __syncthreads();
  }
}

// Leg mode, between the legs' backward and forward launches: the condensed block-tridiagonal
// system of every instance (condensed_solve), one CTA per instance.
__global__ void __launch_bounds__(256) condensed_kernel(const SweepParams p, const int nx) {
  extern __shared__ __align__(16) double smem[];
  BlockDevCtx ctx;
  ctx.tid = threadIdx.x;
  ctx.nthreads = blockDim.x;
  ctx.warp = threadIdx.x >> 5;
  ctx.lane = threadIdx.x & 31;
  ctx.nwarps = blockDim.x >> 5;
  ctx.bar0 = 0;
  ctx.phase = 0;
  for (int inst = blockIdx.x; inst < p.batch; inst += gridDim.x) {
    condensed_solve(ctx, p, nx, inst, smem);
    __syncthreads();
  }
}

// The stage-dense solver (riccati_dense.cuh): one CTA per instance, persistent over the batch.
template <bool PI> __global__ void __launch_bounds__(256) riccati_dense_kernel(const SweepParams p, const DenseDims d) {
  extern __shared__ __align__(16) double smem[];
  BlockDevCtx ctx;
  ctx.tid = threadIdx.x;
  ctx.nthreads = blockDim.x;
  ctx.warp = threadIdx.x >> 5;
  ctx.lane = threadIdx.x & 31;
  ctx.nwarps = blockDim.x >> 5;
  ctx.bar0 = 0;
  ctx.phase = 0;
  for (int inst = blockIdx.x; inst < p.batch; inst += gridDim.x) {
    if constexpr (PI) {
      riccati_dense_sweep(ctx, p, d, inst, smem, InstanceMu());
      flag_bad_mu(p, inst, d.nc > 0 || p.nct > 0, ctx.tid == 0);
    } else {
      riccati_dense_sweep(ctx, p, d, inst, smem);
    }
    __syncthreads();
  }
}

__global__ void collapse_kernel(const SweepParams p, const int nx, const int nu, const int nc) {
  BlockDevCtx ctx;
  ctx.tid = threadIdx.x;
  ctx.nthreads = blockDim.x;
  for (int inst = blockIdx.x; inst < p.batch; inst += gridDim.x)
    collapse_feedback(ctx, p, nx, nu, nc, inst);
}

int block_threads(int nx, int nu, int nc, int nc0, int nth) {
  const BlockDims d = make_block_dims(nx, nu, nc, nc0, nth);
  int need = nx + 1;
  if (d.nk > need)
    need = d.nk;
  if (nx + nc0 > need)
    need = nx + nc0;
  if (d.nr > need)
    need = d.nr;
  if (nth > need)
    need = nth;
  if (need > 256)
    return 0;
  const int nchunk = (d.nt + BLK_CH - 1) / BLK_CH;
  int warps = d.nt * nchunk; // work items of the largest product
  if (warps > 8)
    warps = 8;
  const int wneed = (need + 31) / 32;
  if (warps < wneed)
    warps = wneed;
  return 32 * warps;
}

size_t block_smem_bytes(int nx, int nu, int nc, int nc0, int nth) {
  const BlockDims d = make_block_dims(nx, nu, nc, nc0, nth);
  return (size_t)d.s_end * sizeof(double) + 8 * NBAR;
}

bool block_supported(int nx, int nu, int nc, int nc0, int nth) {
  return block_threads(nx, nu, nc, nc0, nth) > 0 && block_smem_bytes(nx, nu, nc, nc0, nth) <= (size_t)227 * 1024;
}

template <int MAXREG, class D>
static cudaError_t launch_block_t(const SweepParams &p, const D &d, int threads, size_t smem,
                                  cudaStream_t st, int *info) {
  auto kern = p.mueq_b ? riccati_block_kernel<MAXREG, D, true> : riccati_block_kernel<MAXREG, D, false>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess)
    return e;
  e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                           (int)cudaSharedmemCarveoutMaxShared);
  if (e != cudaSuccess)
    return e;
  int nb = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, threads, smem);
  if (e != cudaSuccess)
    return e;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int grid = sms * (nb > 0 ? nb : 1); // persistent CTAs, instances (or legs) strided over them
  const long items = (long)p.batch * (p.legs > 1 ? p.legs : 1);
  if (grid > items)
    grid = (int)items;
  if (info) {
    cudaFuncAttributes fa;
    cudaFuncGetAttributes(&fa, kern);
    info[0] = threads;
    info[1] = (int)smem;
    info[2] = threads;
    info[3] = grid;
    info[4] = fa.numRegs;
    info[5] = nb;
    return cudaSuccess;
  }
  kern<<<grid, threads, smem, st>>>(p, d);
  return cudaGetLastError();
}

// leg mode: the condensed solve of every instance / collapseFeedback
bool condensed_supported(int nx, int nc0, int legs) {
  const int dmax = nx > nc0 ? nx : nc0;
  return legs >= 2 && dmax <= 256 && (size_t)condensed_smem_doubles(nx, nc0, legs) * sizeof(double) <= (size_t)227 * 1024;
}
cudaError_t launch_condensed(const SweepParams &p, int nx, cudaStream_t st) {
  const int dmax = nx > p.nc0 ? nx : p.nc0;
  const int threads = 32 * ((dmax + 31) / 32);
  const size_t smem = (size_t)condensed_smem_doubles(nx, p.nc0, p.legs) * sizeof(double);
  cudaError_t e = cudaFuncSetAttribute(condensed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess)
    return e;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int per_sm = (int)((size_t)227 * 1024 / (smem + 1024));
  per_sm = per_sm < 1 ? 1 : (per_sm > 16 ? 16 : per_sm);
  int grid = sms * per_sm;
  if (grid > p.batch)
    grid = p.batch;
  condensed_kernel<<<grid, threads, smem, st>>>(p, nx);
  return cudaGetLastError();
}
cudaError_t launch_collapse(const SweepParams &p, int nx, int nu, int nc, cudaStream_t st) {
  int grid = p.batch < p.num_sms * 8 ? p.batch : p.num_sms * 8;
  collapse_kernel<<<grid, 128, 0, st>>>(p, nx, nu, nc);
  return cudaGetLastError();
}

static int dense_threads(const DenseDims &d) {
  int need = d.n > d.nx + d.nc0 ? d.n : d.nx + d.nc0;
  if (d.nx + 1 > need)
    need = d.nx + 1;
  return need > 256 ? 0 : 32 * ((need + 31) / 32);
}
bool dense_supported(int nx, int nu, int nc, int nct, int nc0) {
  const DenseDims d = make_dense_dims(nx, nu, nc, nct, nc0);
  return dense_threads(d) > 0 && (size_t)d.s_end * sizeof(double) <= (size_t)227 * 1024;
}
cudaError_t launch_dense(const SweepParams &p, int nx, int nu, int nc, cudaStream_t st) {
  const DenseDims d = make_dense_dims(nx, nu, nc, p.nct, p.nc0);
  const int threads = dense_threads(d);
  const size_t smem = (size_t)d.s_end * sizeof(double);
  auto kern = p.mueq_b ? riccati_dense_kernel<true> : riccati_dense_kernel<false>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess)
    return e;
  int nb = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, threads, smem);
  if (e != cudaSuccess)
    return e;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int grid = sms * (nb > 0 ? nb : 1);
  if (grid > p.batch)
    grid = p.batch;
  kern<<<grid, threads, smem, st>>>(p, d);
  return cudaGetLastError();
}

cudaError_t launch_block(const SweepParams &p, int nx, int nu, int nc, cudaStream_t st, int *info) {
  const BlockDims d = make_block_dims(nx, nu, nc, p.nc0, p.nth, p.legs > 1 ? 0 : -1);
  const int threads = block_threads(nx, nu, nc, p.nc0, p.nth);
  const size_t smem = block_smem_bytes(nx, nu, nc, p.nc0, p.nth);
  // BASELINE config 5 (Talos whole-body walk, nx 57 nu 28, initial condition on the full state):
  // the same code specialised at compile time
  if (nx == 57 && nu == 28 && nc == 0 && p.nc0 == 57 && p.nth == 0 && p.legs <= 1)
    return launch_block_t<255>(p, StaticBlockDims<57, 28, 0, 57>{}, threads, smem, st, info);
  // ... and the reference-faithful Talos dims of SURVEY 0.4 (ndx 56, nu 22)
  if (nx == 56 && nu == 22 && nc == 0 && p.nc0 == 56 && p.nth == 0 && p.legs <= 1)
    return launch_block_t<255>(p, StaticBlockDims<56, 22, 0, 56>{}, threads, smem, st, info);
  // one CTA per SM anyway (shared memory): let it use the whole register file
  if (2 * (smem + 1024) > (size_t)227 * 1024)
    return launch_block_t<255>(p, d, threads, smem, st, info);
  return launch_block_t<128>(p, d, threads, smem, st, info);
}

} // namespace ab2
