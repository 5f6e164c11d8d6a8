// The per-item programs (lq_resolve.cuh, lq_theta.cuh, lq_factor_adjoint.cuh, lq_factor_tangent.cuh) on the host: the
// lanes of one work item are `nl` std::threads that synchronise through a std::barrier, as the lanes of one warp or CTA
// do on the device, and the items run one after another.
#pragma once
#include <barrier>
#include <thread>
#include <vector>

struct EmuCtx {
  int lane, nl;
  std::barrier<> *bar;
  void sync() const { bar->arrive_and_wait(); }
};

// item(ctx) on nl lanes, returning when every lane has finished
template <class F> void run_lanes(int nl, F item) {
  std::barrier<> bar(nl);
  std::vector<std::thread> th;
  for (int l = 0; l < nl; ++l)
    th.emplace_back([&, l] { item(EmuCtx{l, nl, &bar}); });
  for (auto &t : th)
    t.join();
}

// item(ctx, sm, b) for every instance b < batch, on nl lanes and `doubles` of shared memory
template <class F> void run_instances(long batch, int nl, size_t doubles, F item) {
  std::vector<double> sm(doubles);
  for (long b = 0; b < batch; ++b)
    run_lanes(nl, [&](const EmuCtx &ctx) { item(ctx, sm.data(), b); });
}

// item(ctx, sm, b, j0, R) for every instance b < batch and every chunk [j0, j0 + R) of `chunk` of the nrhs columns, on
// nl lanes and `doubles` of shared memory
template <class F> void run_chunks(long batch, int nrhs, int chunk, int nl, size_t doubles, F item) {
  std::vector<double> sm(doubles);
  const int chunks = (nrhs + chunk - 1) / chunk;
  for (long b = 0; b < batch; ++b)
    for (int c = 0; c < chunks; ++c) {
      const int j0 = c * chunk, R = nrhs - j0 < chunk ? nrhs - j0 : chunk;
      run_lanes(nl, [&](const EmuCtx &ctx) { item(ctx, sm.data(), b, j0, R); });
    }
}
