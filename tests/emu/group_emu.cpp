// Host emulation of the CUDA group program (aligator_b200/csrc/riccati_group.cuh):
// a group is G std::threads, sync() is a std::barrier, the TMA bulk copy is a
// memcpy by lane 0.  TEST INFRASTRUCTURE: lets the CPU suite execute the exact
// index arithmetic of the kernel and compare it with the oracle.
#include <barrier>
#include <cstring>
#include <limits>
#include <thread>
#include <vector>

#include "../../aligator_b200/csrc/riccati_configs.h"
#include "../../aligator_b200/csrc/riccati_group.cuh"

namespace {
struct HostCtx {
  int lane;
  int G_; // lanes in the group
  std::barrier<> *bar;
  double *xa, *xb; // fragment exchange for the emulated mma (one slot per lane)
  int *lutp;
  int *cta_ints() const { return lutp; }
  void sync() { bar->arrive_and_wait(); }
  // mma.sync.m8n8k4 f64: lane = 4g+q holds a[g][q], b[q][g], d[g][2q], d[g][2q+1]
  void mma(double (&d)[2], double a, double b) {
    xa[lane] = a;
    xb[lane] = b;
    sync();
    const int g = lane >> 2, q = lane & 3;
    for (int e = 0; e < 2; ++e) {
      double s = 0.0;
      for (int k = 0; k < 4; ++k)
        s += xa[4 * g + k] * xb[4 * (2 * q + e) + k];
      d[e] += s;
    }
    sync();
  }
  double shfl(double v, int src) { // every lane publishes, then reads lane `src`
    xa[lane] = v;
    sync();
    const double r = xa[src];
    sync();
    return r;
  }
  bool all(bool p) {
    xa[lane] = p ? 1.0 : 0.0;
    sync();
    bool r = true;
    for (int l = 0; l < G_; ++l)
      r = r && (xa[l] != 0.0);
    sync();
    return r;
  }
  void issue_copy(int, double *dst, const double *src, int nd) {
    if (lane == 0)
      std::memcpy(dst, src, sizeof(double) * (size_t)nd);
  }
  void copy_expect(int, int) {}
  void copy_add(int, double *dst, const double *src, int nd) {
    if (lane == 0)
      std::memcpy(dst, src, sizeof(double) * (size_t)nd);
  }
  void wait_copy(int) { sync(); }
  void proxy_fence() {}
  void proxy_fence_smem() {}
};

template <class C, class Mu> int run(const ab2::SweepParams &p, const Mu &mu) {
  constexpr int NX = C::NX, G = C::G;
  if (NX + p.nc0 > G)
    return 2;
  for (int inst = 0; inst < p.batch; ++inst) {
    std::vector<double> sm((size_t)C::group_doubles(p.nc0),
                           std::numeric_limits<double>::quiet_NaN());
    std::barrier<> bar(G);
    std::vector<double> xa(G), xb(G);
    std::vector<int> lutv(C::LUT_INTS + 32);
    if constexpr (C::MMA)
      for (int l = 0; l < 32; ++l)
        ab2::fill_mma_lut<C>(lutv.data(), l);
    std::vector<std::thread> th;
    for (int l = 0; l < G; ++l)
      th.emplace_back([&, l] {
        HostCtx ctx{l, G, &bar, xa.data(), xb.data(), lutv.data()};
        ab2::riccati_group_sweep<C>(ctx, p, inst, sm.data(), mu);
      });
    for (auto &t : th)
      t.join();
  }
  return 0;
}

// the mu source as the device launchers pick it: the per-instance array when it is set
template <class C> int run(const ab2::SweepParams &p) {
  return p.mueq_b ? run<C>(p, ab2::InstanceMu()) : run<C>(p, ab2::ScalarMu());
}

// mode 0/1: lane-per-column step, single / double record buffer; 2/3: tensor-core step, double / single.
// PK: Vxx stored packed (every device build) instead of full (the reference the packed program is compared with).
template <int NX, int NU, int NC, int G, bool PK> int dispatch(int mode, const ab2::SweepParams &p) {
  if (mode >= 2) {
    if constexpr (G == 32 && NC == 0 && NX % 2 == 0)
      return mode == 2 ? run<ab2::Cfg<NX, NU, NC, G, true, true, true, PK>>(p)
                       : run<ab2::Cfg<NX, NU, NC, G, false, true, true, PK>>(p);
    else
      return 3;
  }
  return mode ? run<ab2::Cfg<NX, NU, NC, G, true, true, false, PK>>(p)
              : run<ab2::Cfg<NX, NU, NC, G, false, true, false, PK>>(p);
}
} // namespace

extern "C" int emu_stage_record(int nx, int nu, int nc) {
#define X(NX, NU, NC, G)                                                        \
  if (nx == NX && nu == NU && nc == NC)                                         \
    return ab2::Cfg<NX, NU, NC, G>::SREC_PAD;
  AB2_FOR_EACH_CONFIG(X)
#undef X
  return -1;
}

extern "C" int emu_vxx_packed_doubles(int nx) { return ab2::vxx_packed_doubles(nx); }

extern "C" int emu_sweep(int nx, int nu, int nc, int mode, int packed, const ab2::SweepParams *p) {
#define X(NX, NU, NC, G)                                                        \
  if (nx == NX && nu == NU && nc == NC)                                         \
    return packed ? dispatch<NX, NU, NC, G, true>(mode, *p) : dispatch<NX, NU, NC, G, false>(mode, *p);
  AB2_FOR_EACH_CONFIG(X)
#undef X
  return 1;
}
