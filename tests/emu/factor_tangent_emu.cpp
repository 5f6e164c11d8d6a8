// Host emulation of the ab2_gar_factor_tangent program (aligator_b200/csrc/lq_factor_tangent.cuh): each instance runs
// on `nl` std::threads that synchronise through a std::barrier, as the lanes of one warp or CTA do on the device.
// Built by tests/test_factor_tangent_oracle.py with g++ -std=c++20 -pthread.
#include <barrier>
#include <thread>
#include <vector>

#include "../../aligator_b200/csrc/lq_factor_tangent.cuh"

namespace {
struct EmuCtx {
  int lane, nl;
  std::barrier<> *bar;
  void sync() const { bar->arrive_and_wait(); }
};
} // namespace

// dims: batch, N, nx, nu, nc, nct, nc0, srec, trec, stage_head, lanes
// in:   stage, term, fb, fbT, Vxx, Vxx0, ff, vx, ffT, d_stage, d_term
// out:  ff, fb, vxx, vx, fft, fbt (tangents; null = not written)
extern "C" int emu_factor_tangent(const int *dims, double mueq, const double *mueq_b, const double *const *in,
                                  double *const *out) {
  ab2::FactorTangentArgs a{};
  ab2::ResolveArgs &r = a.fac;
  r.batch = dims[0], r.N = dims[1], r.nx = dims[2], r.nu = dims[3], r.nc = dims[4], r.nct = dims[5], r.nc0 = dims[6];
  r.srec = dims[7], r.trec = dims[8], r.stage_head = dims[9];
  const int nl = dims[10];
  r.stage = in[0], r.term = in[1], r.fb = in[2], r.fbT = in[3], r.Vxx = in[4], r.Vxx0 = in[5];
  a.ff = in[6], a.vx = in[7], a.ffT = in[8];
  a.d_stage = in[9], a.d_term = in[10];
  a.o_ff = out[0], a.o_fb = out[1], a.o_vxx = out[2], a.o_vx = out[3], a.o_fft = out[4], a.o_fbt = out[5];
  r.mueq = mueq;
  r.mueq_b = mueq_b;
  std::vector<double> sm(ab2::factor_tangent_item_doubles(r.nx, r.nu, r.nc));
  for (long b = 0; b < r.batch; ++b) {
    std::barrier<> bar(nl);
    std::vector<std::thread> th;
    for (int l = 0; l < nl; ++l)
      th.emplace_back([&, l] { ab2::factor_tangent_item(a, EmuCtx{l, nl, &bar}, sm.data(), b); });
    for (auto &t : th)
      t.join();
  }
  return 0;
}

// Every shape `supported` (the library's ab2_gar_supported) accepts with nx, nu, nc < lim and nc0 in {0, 1, nx/2, nx}:
// how many are accepted (*accepted), how many of those need more than 227 KB of shared memory (the return value; the
// first one in *bad = nx, nu, nc, nc0), and the largest item that fits, in bytes (*largest).
extern "C" long emu_factor_tangent_size_scan(int (*supported)(int, int, int, int), int lim, int *bad, long *largest,
                                             long *accepted) {
  long over = 0;
  *largest = 0;
  *accepted = 0;
  for (int nx = 1; nx < lim; ++nx)
    for (int nu = 1; nu < lim; ++nu)
      for (int nc = 0; nc < lim; ++nc) {
        const int nc0s[4] = {0, 1, nx / 2, nx};
        for (int i = 0; i < 4; ++i) {
          const int nc0 = nc0s[i];
          if (i && nc0 == nc0s[i - 1])
            continue;
          if (!supported(nx, nu, nc, nc0))
            continue;
          ++*accepted;
          const long bytes = (long)ab2::factor_tangent_item_doubles(nx, nu, nc) * (long)sizeof(double);
          if (bytes > 227 * 1024) {
            if (over++ == 0)
              bad[0] = nx, bad[1] = nu, bad[2] = nc, bad[3] = nc0;
          } else if (bytes > *largest) {
            *largest = bytes;
          }
        }
      }
  return over;
}

extern "C" long emu_factor_tangent_item_bytes(int nx, int nu, int nc) {
  return (long)ab2::factor_tangent_item_doubles(nx, nu, nc) * (long)sizeof(double);
}
