// Host emulation of the sweep programs with a per-instance mu (ab2::InstanceMu, the mu source of the *_v launches):
// the warp-per-instance group program (packed-Vxx builds, both step implementations), the CTA-per-instance program,
// its leg mode and the stage-dense program.  TEST INFRASTRUCTURE (see group_emu.cpp, block_emu.cpp).
//
// The Python side passes its ctypes copy of SweepParams, which ends before SweepParams::mueq_b, with its size; the
// harness copies that prefix into a full, zero-initialised SweepParams of its own and sets mueq_b there.  The existing
// harness entry points and their parameter structs are untouched.
#include <cstddef>

#include "block_emu.cpp"
#include "group_packed_emu.cpp"

namespace {
// A full SweepParams from the caller's prefix of `bytes` bytes, with mueq_b = mu; nullptr-equivalent (batch = -1) when
// the prefix would reach into mueq_b.
ab2::SweepParams local_params(const void *pp, size_t bytes, const double *mu) {
  ab2::SweepParams q;
  std::memset(&q, 0, sizeof(q));
  if (bytes > offsetof(ab2::SweepParams, mueq_b)) {
    q.batch = -1;
    return q;
  }
  std::memcpy(&q, pp, bytes);
  q.mueq_b = mu;
  return q;
}

template <class C> int run_pi(const ab2::SweepParams &p) {
  constexpr int NX = C::NX, G = C::G;
  if (NX + p.nc0 > G)
    return 2;
  for (int inst = 0; inst < p.batch; ++inst) {
    std::vector<double> sm((size_t)C::group_doubles(p.nc0), std::numeric_limits<double>::quiet_NaN());
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
        ab2::riccati_group_sweep<C>(ctx, p, inst, sm.data(), ab2::InstanceMu());
      });
    for (auto &t : th)
      t.join();
  }
  return 0;
}

// mode 0/1: lane-per-column step, single / double record buffer; 2/3: tensor-core step, double / single
template <int NX, int NU, int NC, int G> int dispatch_pi(int mode, const ab2::SweepParams &p) {
  if (mode >= 2) {
    if constexpr (G == 32 && NC == 0 && NX % 2 == 0)
      return mode == 2 ? run_pi<ab2::Cfg<NX, NU, NC, G, true, true, true, true>>(p)
                       : run_pi<ab2::Cfg<NX, NU, NC, G, false, true, true, true>>(p);
    else
      return 3;
  }
  return mode ? run_pi<ab2::Cfg<NX, NU, NC, G, true, true, false, true>>(p)
              : run_pi<ab2::Cfg<NX, NU, NC, G, false, true, false, true>>(p);
}

template <class D> int run_block_pi(const D &d, int nwarps, const ab2::SweepParams &p) {
  const int nx = d.nx;
  const int T = 32 * nwarps;
  if (nx + 1 > T || d.nk > T || nx + p.nc0 > T || d.nr > T || d.nth > T)
    return 2;
  const int legs = p.legs > 1 ? p.legs : 1;
  for (int item = 0; item < p.batch * legs; ++item)
    run_cta(nwarps, (size_t)d.s_end, [&](HostBlockCtx &ctx, double *sm) {
      ab2::riccati_block_sweep(ctx, p, d, item / legs, sm, item % legs, ab2::InstanceMu());
    });
  return 0;
}
} // namespace

extern "C" int emu_pi_params_offset() { return (int)offsetof(ab2::SweepParams, mueq_b); }

extern "C" int emu_pi_sweep(int nx, int nu, int nc, int mode, const void *pp, long bytes, const double *mu) {
  const ab2::SweepParams p = local_params(pp, (size_t)bytes, mu);
  if (p.batch < 0)
    return 4;
#define X(NX, NU, NC, G)                                                        \
  if (nx == NX && nu == NU && nc == NC)                                         \
    return dispatch_pi<NX, NU, NC, G>(mode, p);
  AB2_FOR_EACH_CONFIG(X)
#undef X
  return 1;
}

extern "C" int emu_pi_block_sweep(int nx, int nu, int nc, int nwarps, const void *pp, long bytes, const double *mu) {
  const ab2::SweepParams p = local_params(pp, (size_t)bytes, mu);
  if (p.batch < 0)
    return 4;
  return run_block_pi(ab2::make_block_dims(nx, nu, nc, p.nc0), nwarps, p);
}

// leg mode: legs backward -> condensed solve -> legs forward, as emu_block_legs (mode 3) does it
extern "C" int emu_pi_block_legs(int nx, int nu, int nc, int nwarps, const void *pp, long bytes, const double *mu) {
  ab2::SweepParams p = local_params(pp, (size_t)bytes, mu);
  if (p.batch < 0)
    return 4;
  if (p.legs < 2 || p.N + 1 < p.legs)
    return 3;
  p.nth = nx;
  const ab2::BlockDims d = ab2::make_block_dims(nx, nu, nc, p.nc0, nx, 0);
  for (int b = 0; b < p.batch; ++b) {
    p.status[b] = 0;
    if (p.pivstat)
      p.pivstat[b] = 0;
  }
  p.do_bwd = 1;
  p.do_fwd = 0;
  if (int rc = run_block_pi(d, nwarps, p))
    return rc;
  const int dmax = nx > p.nc0 ? nx : p.nc0;
  for (int b = 0; b < p.batch; ++b)
    run_cta((dmax + 31) / 32, (size_t)ab2::condensed_smem_doubles(nx, p.nc0, p.legs),
            [&](HostBlockCtx &ctx, double *sm) { ab2::condensed_solve(ctx, p, nx, b, sm); });
  p.do_bwd = 0;
  p.do_fwd = 1;
  return run_block_pi(d, nwarps, p);
}

extern "C" int emu_pi_dense_sweep(int nx, int nu, int nc, int nwarps, const void *pp, long bytes, const double *mu) {
  const ab2::SweepParams p = local_params(pp, (size_t)bytes, mu);
  if (p.batch < 0)
    return 4;
  const ab2::DenseDims d = ab2::make_dense_dims(nx, nu, nc, p.nct, p.nc0);
  const int T = 32 * nwarps;
  if (d.n > T || nx + p.nc0 > T || nx + 1 > T)
    return 2;
  for (int inst = 0; inst < p.batch; ++inst)
    run_cta(nwarps, (size_t)d.s_end, [&](HostBlockCtx &ctx, double *sm) {
      ab2::riccati_dense_sweep(ctx, p, d, inst, sm, ab2::InstanceMu());
    });
  return 0;
}
