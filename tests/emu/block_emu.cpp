// Host emulation of the CTA-per-instance sweep (aligator_b200/csrc/riccati_block.cuh):
// a CTA is 32*NW std::threads, sync() is a CTA-wide std::barrier, the warp-wide mma is
// a fragment exchange behind a per-warp barrier, the TMA bulk copy is a memcpy by
// thread 0.  TEST INFRASTRUCTURE (see group_emu.cpp).
#include <barrier>
#include <cstring>
#include <limits>
#include <memory>
#include <thread>
#include <vector>

#include "../../aligator_b200/csrc/riccati_block.cuh"
#include "../../aligator_b200/csrc/riccati_dense.cuh"

namespace {
struct HostBlockCtx {
  int tid, nthreads, warp, lane, nwarps;
  std::barrier<> *cta;
  std::barrier<> **sub; // sub[w-1]: barrier over the first w warps
  std::barrier<> *wbar;
  double *xa, *xb; // this warp's exchange slots
  void sync() { cta->arrive_and_wait(); }
  int *orflag; // shared by the CTA's threads
  int sync_or(int v) {
    if (v)
      __atomic_store_n(orflag, 1, __ATOMIC_SEQ_CST);
    cta->arrive_and_wait();
    const int r = __atomic_load_n(orflag, __ATOMIC_SEQ_CST);
    cta->arrive_and_wait();
    if (tid == 0)
      *orflag = 0;
    cta->arrive_and_wait();
    return r;
  }
  void sync_sub(int nth) { sub[nth / 32 - 1]->arrive_and_wait(); }
  void mma(double (&d)[2], double a, double b) {
    xa[lane] = a;
    xb[lane] = b;
    wbar->arrive_and_wait();
    const int g = lane >> 2, q = lane & 3;
    for (int e = 0; e < 2; ++e) {
      double s = 0.0;
      for (int k = 0; k < 4; ++k)
        s += xa[4 * g + k] * xb[4 * (2 * q + e) + k];
      d[e] += s;
    }
    wbar->arrive_and_wait();
  }
  void wsync() { wbar->arrive_and_wait(); }
  void atomic_or(int *q, int v) { *q |= v; }   // (the emulation runs the work items one after another)
  void atomic_add(int *q, int v) { *q += v; }
  double shfl(double v, int src) {
    xa[lane] = v;
    wbar->arrive_and_wait();
    const double r = xa[src & 31];
    wbar->arrive_and_wait();
    return r;
  }
  bool all(bool p) {
    xb[lane] = p ? 1.0 : 0.0;
    wbar->arrive_and_wait();
    bool r = true;
    for (int i = 0; i < 32; ++i)
      r = r && (xb[i] != 0.0);
    wbar->arrive_and_wait();
    return r;
  }
  void issue_copy(int, double *dst, const double *src, int nd) {
    if (tid == 0)
      std::memcpy(dst, src, sizeof(double) * (size_t)nd);
  }
  void wait_copy(int) { sync(); }
  void proxy_fence() {}
};
} // namespace

// nth > 0: parametric records
extern "C" int emu_block_stage_record(int nx, int nu, int nc, int nth) {
  return ab2::make_block_dims(nx, nu, nc, 0, nth).srec_pad;
}

template <class D> static int run_block(const D &d, int nwarps, const ab2::SweepParams &p);
template <class F> static void run_cta(int nwarps, size_t smem_doubles, F body);

// run-time dimensions; parametric problems when p->nth > 0
extern "C" int emu_block_sweep(int nx, int nu, int nc, int nwarps, const ab2::SweepParams *p) {
  return run_block(ab2::make_block_dims(nx, nu, nc, p->nc0, p->nth), nwarps, *p);
}

// the compile-time specialisation (StaticBlockDims) of two small shapes, to execute that
// instantiation of the code on the CPU
extern "C" int emu_block_sweep_static(int nx, int nu, int nc, int nwarps, const ab2::SweepParams *p) {
  if (nx == 7 && nu == 3 && nc == 0 && p->nc0 == 7)
    return run_block(ab2::StaticBlockDims<7, 3, 0, 7>{}, nwarps, *p);
  if (nx == 9 && nu == 5 && nc == 3 && p->nc0 == 9)
    return run_block(ab2::StaticBlockDims<9, 5, 3, 9>{}, nwarps, *p);
  return 1;
}

// one emulated CTA of 32*nwarps threads running body(ctx, smem)
template <class F> static void run_cta(int nwarps, size_t smem_doubles, F body) {
  const int T = 32 * nwarps;
  std::vector<double> sm(smem_doubles, std::numeric_limits<double>::quiet_NaN());
  std::barrier<> cta(T);
  std::vector<std::unique_ptr<std::barrier<>>> wb;
  for (int w = 0; w < nwarps; ++w)
    wb.emplace_back(new std::barrier<>(32));
  std::vector<std::unique_ptr<std::barrier<>>> subs;
  std::vector<std::barrier<> *> subp;
  for (int w = 1; w <= nwarps; ++w) {
    subs.emplace_back(new std::barrier<>(32 * w));
    subp.push_back(subs.back().get());
  }
  std::vector<double> xa(T), xb(T);
  int orflag = 0;
  std::vector<std::thread> th;
  for (int t = 0; t < T; ++t)
    th.emplace_back([&, t] {
      HostBlockCtx ctx{t, T, t / 32, t % 32, nwarps, &cta, subp.data(), wb[t / 32].get(),
                       xa.data() + 32 * (t / 32), xb.data() + 32 * (t / 32), &orflag};
      body(ctx, sm.data());
    });
  for (auto &t : th)
    t.join();
}

template <class D, class Mu> static int run_block(const D &d, int nwarps, const ab2::SweepParams &p, const Mu &mu) {
  const int nx = d.nx;
  const int T = 32 * nwarps;
  if (nx + 1 > T || d.nk > T || nx + p.nc0 > T || d.nr > T || d.nth > T)
    return 2;
  const int legs = p.legs > 1 ? p.legs : 1;
  for (int item = 0; item < p.batch * legs; ++item)
    run_cta(nwarps, (size_t)d.s_end,
            [&](HostBlockCtx &ctx, double *sm) { ab2::riccati_block_sweep(ctx, p, d, item / legs, sm, item % legs, mu); });
  return 0;
}

// the mu source as the device launchers pick it: the per-instance array when it is set
template <class D> static int run_block(const D &d, int nwarps, const ab2::SweepParams &p) {
  return p.mueq_b ? run_block(d, nwarps, p, ab2::InstanceMu()) : run_block(d, nwarps, p, ab2::ScalarMu());
}

// Leg mode (gar::ParallelRiccatiSolver): legs backward -> condensed solve -> legs forward, as the
// three launches of the product do it.  mode bit 0: backward + condensed, bit 1: forward, bit 2: collapseFeedback
extern "C" int emu_block_legs(int nx, int nu, int nc, int nwarps, int mode, const ab2::SweepParams *pp) {
  ab2::SweepParams p = *pp;
  if (p.legs < 2 || p.N + 1 < p.legs)
    return 3;
  p.nth = nx;
  const ab2::BlockDims d = ab2::make_block_dims(nx, nu, nc, p.nc0, nx, 0);
  if (mode & 1) {
    for (int b = 0; b < p.batch; ++b) {
      p.status[b] = 0;
      if (p.pivstat)
        p.pivstat[b] = 0;
    }
    p.do_bwd = 1;
    p.do_fwd = 0;
    if (int rc = run_block(d, nwarps, p))
      return rc;
    const int dmax = nx > p.nc0 ? nx : p.nc0;
    for (int b = 0; b < p.batch; ++b)
      run_cta((dmax + 31) / 32, (size_t)ab2::condensed_smem_doubles(nx, p.nc0, p.legs),
              [&](HostBlockCtx &ctx, double *sm) { ab2::condensed_solve(ctx, p, nx, b, sm); });
  }
  if (mode & 4)
    for (int b = 0; b < p.batch; ++b)
      run_cta(1, 2, [&](HostBlockCtx &ctx, double *) { ab2::collapse_feedback(ctx, p, nx, nu, nc, b); });
  if (mode & 2) {
    p.do_bwd = 0;
    p.do_fwd = 1;
    if (int rc = run_block(d, nwarps, p))
      return rc;
  }
  return 0;
}

// The stage-dense solver (riccati_dense.cuh) on emulated CTAs.
template <class Mu> static int run_dense(int nx, int nu, int nc, int nwarps, const ab2::SweepParams &p, const Mu &mu) {
  const ab2::DenseDims d = ab2::make_dense_dims(nx, nu, nc, p.nct, p.nc0);
  const int T = 32 * nwarps;
  if (d.n > T || nx + p.nc0 > T || nx + 1 > T)
    return 2;
  for (int inst = 0; inst < p.batch; ++inst)
    run_cta(nwarps, (size_t)d.s_end, [&](HostBlockCtx &ctx, double *sm) { ab2::riccati_dense_sweep(ctx, p, d, inst, sm, mu); });
  return 0;
}

extern "C" int emu_dense_sweep(int nx, int nu, int nc, int nwarps, const ab2::SweepParams *p) {
  return p->mueq_b ? run_dense(nx, nu, nc, nwarps, *p, ab2::InstanceMu()) : run_dense(nx, nu, nc, nwarps, *p, ab2::ScalarMu());
}
