// riccati_launch.cuh -- device execution context, the persistent sweep kernel and
// its launch variants.  Included by kernel_inst.cu (one translation unit per
// compile-time shape, built in parallel) and by gar_cuda.cu (the C ABI).
#pragma once
#include <cuda_runtime.h>

#include "riccati_group.cuh"

namespace ab2 {

// ---------------------------------------------------------------------------
// Device execution context of one group.
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

constexpr int NBAR = 8; // mbarriers per group (backward uses 2, the forward ring up to 8)

template <int G, bool TMA> struct DevCtx {
  int lane;
  unsigned mask;
  uint32_t bar0; // shared address of this group's NBAR mbarriers
  uint32_t phase; // bit p = parity to wait for on barrier p
  int *cta_lut;   // per-CTA scratch for per-lane constants (tensor-core step)
  __device__ __forceinline__ int *cta_ints() const { return cta_lut; }

  __device__ __forceinline__ void sync() { __syncwarp(mask); }
  // value of `v` in lane `src` of this group / vote over the group
  __device__ __forceinline__ double shfl(double v, int src) { return __shfl_sync(mask, v, src, G); }
  __device__ __forceinline__ bool all(bool p) { return __all_sync(mask, p); }

  // D(8x8) += A(8x4) B(4x8) on the FP64 tensor cores (SASS: DMMA.884); full warp only.
  __device__ __forceinline__ void mma(double (&d)[2], double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(d[0]), "+d"(d[1])
                 : "d"(a), "d"(b));
  }

  __device__ __forceinline__ void init(uint64_t *bars) {
    bar0 = smem_u32(bars);
    phase = 0;
    if (TMA) {
      if (lane == 0) {
        for (int b = 0; b < NBAR; ++b)
          asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar0 + 8 * b));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      }
    }
    __syncwarp(mask);
  }

  // Stage `nd` doubles (nd even, 16-byte aligned both sides) global -> shared.
  __device__ __forceinline__ void issue_copy(int part, double *dst, const double *src, int nd) {
    if (TMA) {
      if (lane == 0) {
        const uint32_t bar = bar0 + 8 * part;
        const uint32_t bytes = (uint32_t)nd * 8u;
        // Ordering against the generic proxy: a refill of a buffer that was only READ through
        // the generic proxy needs no proxy fence (the reads completed before the group
        // synchronisation that precedes this call -- the consumer-release pattern).  Every
        // place where lanes WROTE through the generic proxy what a bulk copy later overwrites
        // (stashed columns in the record buffer, the initial-stage workspace under the forward
        // ring) or reads (ff / fb / Vxx / vx in global memory, re-read by the fused forward)
        // executes proxy_fence() in the writing lanes before that synchronisation.
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
                     : "memory");
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                smem_u32(dst)),
            "l"(src), "r"(bytes), "r"(bar)
            : "memory");
      }
    } else {
      const uint32_t d = smem_u32(dst);
      for (int c = lane; c < nd / 2; c += G)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + 16u * c), "l"(src + 2 * c)
                     : "memory");
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
  }

  // Several bulk copies completing on ONE barrier phase: announce the total, then add the pieces.
  __device__ __forceinline__ void copy_expect(int part, int nd_total) {
    if (TMA) {
      if (lane == 0)
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar0 + 8 * part),
                     "r"((uint32_t)nd_total * 8u)
                     : "memory");
    }
  }
  __device__ __forceinline__ void copy_add(int part, double *dst, const double *src, int nd) {
    if (TMA) {
      if (lane == 0)
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                smem_u32(dst)),
            "l"(src), "r"((uint32_t)nd * 8u), "r"(bar0 + 8 * part)
            : "memory");
    } else {
      const uint32_t d = smem_u32(dst);
      for (int c = lane; c < nd / 2; c += G)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + 16u * c), "l"(src + 2 * c)
                     : "memory");
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
  }

  // Every lane that wrote (through the generic proxy) shared memory a bulk store will read
  // calls this BEFORE the group synchronisation that precedes bulk_store().
  __device__ __forceinline__ void async_fence() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
  // Generic-proxy writes of this lane (shared AND global) ordered before later async-proxy
  // (TMA) accesses: executed by every writing lane before the synchronisation that precedes
  // the bulk copy which overwrites or reads what it wrote (PTX memory model, proxies).
  __device__ __forceinline__ void proxy_fence() { asm volatile("fence.proxy.async;" ::: "memory"); }
  __device__ __forceinline__ void proxy_fence_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
  // Shared -> global bulk store of `nd` doubles (TMA).  One lane issues.
  __device__ __forceinline__ void bulk_store(double *gdst, const double *ssrc, int nd) {
    if (lane == 0) {
      asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
                   "r"(smem_u32(ssrc)), "r"((uint32_t)nd * 8u)
                   : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
  }
  // the source of every earlier bulk_store may be overwritten after this + a sync
  __device__ __forceinline__ void bulk_store_wait_read() {
    if (lane == 0)
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
  }

  __device__ __forceinline__ void wait_copy(int part) {
    if (TMA) {
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
    } else {
      asm volatile("cp.async.wait_all;" ::: "memory");
    }
    __syncwarp(mask);
  }
};

// ---------------------------------------------------------------------------
// The persistent sweep kernel: every group walks the whole horizon of its
// instance (backward, initial stage, forward) inside one launch.
// ---------------------------------------------------------------------------
// PI: per-instance mu (SweepParams::mueq_b, the *_v launches); false = the scalar p.mueq
template <class C, int WARPS, int MAXREG, bool TMA, bool PI>
__global__ void __launch_bounds__(WARPS * 32) __maxnreg__(MAXREG)
    riccati_sweep_kernel(const SweepParams p, const int group_doubles) {
  extern __shared__ __align__(16) double smem[];
  constexpr int IPW = 32 / C::G; // instances per warp
  const int warp = threadIdx.x >> 5;
  const int lane32 = threadIdx.x & 31;
  const int gsub = lane32 / C::G;
  const int group_in_cta = warp * IPW + gsub;
  const int inst = blockIdx.x * (WARPS * IPW) + group_in_cta;
  if constexpr (C::MMA) { // the per-CTA table of per-lane constants: one writer, then a CTA barrier
    fill_mma_lut<C>(reinterpret_cast<int *>(smem + (size_t)(WARPS * IPW) * group_doubles + (size_t)(WARPS * IPW) * NBAR),
                    lane32, warp, WARPS);
    __syncthreads();
  }
  if (inst >= p.batch)
    return; // whole group leaves together
  double *sm = smem + (size_t)group_in_cta * group_doubles;
  uint64_t *bars =
      reinterpret_cast<uint64_t *>(smem + (size_t)(WARPS * IPW) * group_doubles) + NBAR * group_in_cta;
  DevCtx<C::G, TMA> ctx;
  ctx.cta_lut = reinterpret_cast<int *>(smem + (size_t)(WARPS * IPW) * group_doubles + (size_t)(WARPS * IPW) * NBAR);
  ctx.lane = lane32 % C::G;
  ctx.mask = (C::G == 32) ? 0xffffffffu : (((1u << C::G) - 1u) << (gsub * C::G));
  ctx.init(bars);
  if (p.stagger_ns > 0) { // resident slot of this warp on its SM (first wave: CTA b runs on SM b mod num_sms)
    const int slot = (blockIdx.x / p.num_sms) * WARPS + warp;
    __nanosleep((unsigned)(slot * p.stagger_ns));
  }
  if constexpr (PI) {
    riccati_group_sweep<C>(ctx, p, inst, sm, InstanceMu());
    flag_bad_mu(p, inst, C::NC > 0 || p.nct > 0, ctx.lane == 0);
  } else {
    riccati_group_sweep<C>(ctx, p, inst, sm);
  }
}

// ---------------------------------------------------------------------------
// Shape dispatch.
// ---------------------------------------------------------------------------
struct KernelEntry {
  int nx, nu, nc, G;
  int srec_pad;
  void (*group_doubles)(int nc0, int gd[4]);
  cudaError_t (*launch)(const SweepParams &, int variant, const int gd[4], cudaStream_t, int *info);
};

template <class C, int WARPS, int MAXREG, bool TMA>
inline cudaError_t launch_one(const SweepParams &p, int gd, cudaStream_t st, int *info) {
  constexpr int IPW = 32 / C::G;
  const int groups = WARPS * IPW;
  size_t smem = (size_t)groups * gd * sizeof(double) + (size_t)groups * 8 * NBAR + (size_t)C::LUT_INTS * 4;
  // the per-instance instantiation serves the *_v launches; occupancy and launch shape are decided alike
  auto kern = p.mueq_b ? riccati_sweep_kernel<C, WARPS, MAXREG, TMA, true> : riccati_sweep_kernel<C, WARPS, MAXREG, TMA, false>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess)
    return e;
  // the sweep lives in shared memory: ask for the largest carve-out (227 KB per SM)
  e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                           (int)cudaSharedmemCarveoutMaxShared);
  if (e != cudaSuccess)
    return e;
  const int grid = (p.batch + groups - 1) / groups;
  // Residency.  The SM saturates below its maximum residency (taken as 12 resident warps
  // below), so extra resident CTAs only slow each other down; what costs is a partly filled
  // LAST round.  Keep the smallest residency that still needs the minimum number of rounds,
  // enforced by padding the dynamic shared-memory request (the system reserves 1 KB per CTA).
  // (C2 on 132 SMs: 8 CTAs/SM = rounds of 2112 + 1984 instances; 7 would need a third round.)
  // p.ctas_per_sm > 0 overrides, < 0 keeps the maximum.
  {
    static thread_local size_t cached_smem[2] = {0, 0}; // per kernel instantiation
    static thread_local int cached_cmax[2] = {0, 0};
    const int ci = p.mueq_b ? 1 : 0;
    if (cached_smem[ci] != smem) {
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cached_cmax[ci], kern, WARPS * 32, smem);
      if (e != cudaSuccess)
        return e;
      cached_smem[ci] = smem;
    }
    const int cmax = cached_cmax[ci];
    int want = p.ctas_per_sm;
    if (want == 0 && cmax > 1) {
      const int sms = p.num_sms > 0 ? p.num_sms : 132;
      auto rounds = [&](int c) { return (grid + sms * c - 1) / (sms * c); };
      want = cmax;
      while ((want - 1) * WARPS >= 12 && rounds(want - 1) == rounds(cmax))
        --want; // (never below 12 resident warps: under that the SM is not saturated)
    }
    if (want > 0 && want < cmax) {
      const size_t pad = (((size_t)227 * 1024 / want) - 1024) & ~(size_t)15;
      if (pad > smem) {
        smem = pad;
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess)
          return e;
      }
    }
  }
  if (info) {
    cudaFuncAttributes fa;
    cudaFuncGetAttributes(&fa, kern);
    info[0] = C::G;
    info[1] = (int)smem;
    info[2] = WARPS * 32;
    info[3] = grid;
    info[4] = fa.numRegs;
    int nb = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, WARPS * 32, smem);
    info[5] = nb;
    return cudaSuccess;
  }
  kern<<<grid, WARPS * 32, smem, st>>>(p, gd);
  return cudaGetLastError();
}

// Launch variants per shape (ab2_gar_tuning.variant); -1 = automatic:
//   the tensor-core variant 7 where the shape allows it (full warp per instance, nc = 0,
//   even nx), else variant 6.
//   0: lane-per-column step, 2 warps/CTA, <= 144 registers, double-buffered records, TMA
//   1: lane-per-column, 4 warps/CTA x 7 CTAs/SM (<= 72 registers), single record buffer, TMA
//   2: as 0 with cp.async (LDGSTS) staging instead of TMA
//   3: as 1 with cp.async staging
//   4: as 1 with the cooperative shared-memory Bunch-Kaufman
//   5: as 0 with the cooperative shared-memory Bunch-Kaufman
//   6: as 0 capped at 128 registers (8 CTAs = 16 warps per SM)
//   7: stage step on the FP64 tensor cores (DMMA m8n8k4), 128 registers, 16 warps per SM
//   8: as 7 with 168 registers (12 warps per SM, no spills)
//  10: as 7 with a single record buffer refilled in two parts (smallest shared-memory footprint)
template <int NX, int NU, int NC, int G>
inline cudaError_t launch_cfg(const SweepParams &p, int variant, const int gd[4], cudaStream_t st, int *info) {
  // every device build stores Vxx packed (vxx_layout.h)
  using CS = Cfg<NX, NU, NC, G, false, true, false, true>;
  using CD = Cfg<NX, NU, NC, G, true, true, false, true>;
  if (variant < 0) {
    variant = 6;
    if constexpr (G == 32 && NC == 0 && NX % 2 == 0) {
      // Tensor-core builds.  What decides is the number of ROUNDS the batch needs:
      //   7: double-buffered records, 128 registers (<= 8 CTAs/SM)
      //   8: double-buffered records, 168 registers, no spills (<= 6 CTAs/SM)
      //  10: single record buffer, 128 registers: the smallest footprint (<= 8 CTAs/SM)
      // fewest rounds wins; ties go to 7 when it reaches 8 CTAs/SM, else 8, else 10.
      using CM = Cfg<NX, NU, NC, G, true, true, true, true>;
      const int sms = p.num_sms > 0 ? p.num_sms : 132;
      const int grid = (p.batch + 1) / 2;
      auto ctas = [&](int gdw, int cap) {
        const size_t smem = (size_t)2 * gdw * sizeof(double) + 2 * 8 * NBAR + (size_t)CM::LUT_INTS * 4;
        const int c = (int)((size_t)227 * 1024 / (smem + 1024));
        return c < cap ? (c < 1 ? 1 : c) : cap;
      };
      auto rounds = [&](int c) { return (grid + sms * c - 1) / (sms * c); };
      const int c7 = ctas(gd[2], 8), c8 = ctas(gd[2], 6), c10 = ctas(gd[3], 8);
      const int r7 = rounds(c7), r8 = rounds(c8), r10 = rounds(c10);
      if (c7 == 8 && r7 <= r8 && r7 <= r10)
        variant = 7;
      else if (r8 <= r7 && r8 <= r10)
        variant = 8;
      else if (r10 < r7)
        variant = 10;
      else
        variant = 7;
    }
  }
  if (variant == 1)
    return launch_one<CS, 4, 72, true>(p, gd[0], st, info);
  if (variant == 2)
    return launch_one<CD, 2, 144, false>(p, gd[1], st, info);
  if (variant == 3)
    return launch_one<CS, 4, 72, false>(p, gd[0], st, info);
  if (variant == 4)
    return launch_one<Cfg<NX, NU, NC, G, false, false, false, true>, 4, 72, true>(p, gd[0], st, info);
  if (variant == 5)
    return launch_one<Cfg<NX, NU, NC, G, true, false, false, true>, 2, 144, true>(p, gd[1], st, info);
  if (variant == 6) // as 0 capped at 128 registers (8 CTAs/SM)
    return launch_one<CD, 2, 128, true>(p, gd[1], st, info);
  if constexpr (G == 32 && NC == 0 && NX % 2 == 0) {
    using CM = Cfg<NX, NU, NC, G, true, true, true, true>;
    if (variant == 7) // stage step on the FP64 tensor cores (DMMA), 2 warps/CTA
      return launch_one<CM, 2, 128, true>(p, gd[2], st, info);
    if (variant == 8) // same, 168 registers
      return launch_one<CM, 2, 168, true>(p, gd[2], st, info);
    if (variant == 10) // same as 7 with a single record buffer refilled in two parts
      return launch_one<Cfg<NX, NU, NC, G, false, true, true, true>, 2, 128, true>(p, gd[3], st, info);
  }
  return launch_one<CD, 2, 144, true>(p, gd[1], st, info);
}
template <int NX, int NU, int NC, int G> inline void group_doubles_cfg(int nc0, int gd[4]) {
  gd[0] = Cfg<NX, NU, NC, G, false, true, false, true>::group_doubles(nc0);
  gd[1] = Cfg<NX, NU, NC, G, true, true, false, true>::group_doubles(nc0);
  gd[2] = gd[1];
  gd[3] = gd[0];
  if constexpr (G == 32 && NC == 0 && NX % 2 == 0) {
    gd[2] = Cfg<NX, NU, NC, G, true, true, true, true>::group_doubles(nc0);
    gd[3] = Cfg<NX, NU, NC, G, false, true, true, true>::group_doubles(nc0);
  }
}

} // namespace ab2
