// Lanes of one work item of the per-item programs (lq_resolve.cuh, lq_factor_adjoint.cuh, lq_factor_tangent.cuh) on
// the host: `nl` std::threads that synchronise through a std::barrier, as the lanes of one warp or CTA do on the device.
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
