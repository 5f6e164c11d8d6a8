// Host emulation of the ab2_gar_factor_adjoint program (aligator_b200/csrc/lq_factor_adjoint.cuh): each instance runs
// on `nl` emulated lanes (item_emu.h).  Part of the emulation library (emu.cpp).
#include "../../aligator_b200/csrc/lq_factor_adjoint.cuh"
#include "item_emu.h"

// dims: batch, N, nx, nu, nc, nct, nc0, srec, trec, stage_head, lanes
// in:   stage, term, fb, fbT, Vxx, Vxx0, ff, vx, ffT, c_ff, c_fb, c_vxx, c_vx, c_fft, c_fbt
// out:  g_stage, g_term, g_G0, g_g0
extern "C" int emu_factor_adjoint(const int *dims, double mueq, const double *mueq_b, const double *const *in,
                                  double *const *out) {
  ab2::FactorAdjointArgs a{};
  ab2::ResolveArgs &r = a.fac;
  r.batch = dims[0], r.N = dims[1], r.nx = dims[2], r.nu = dims[3], r.nc = dims[4], r.nct = dims[5], r.nc0 = dims[6];
  r.srec = dims[7], r.trec = dims[8], r.stage_head = dims[9];
  const int nl = dims[10];
  r.stage = in[0], r.term = in[1], r.fb = in[2], r.fbT = in[3], r.Vxx = in[4], r.Vxx0 = in[5];
  a.ff = in[6], a.vx = in[7], a.ffT = in[8];
  a.c_ff = in[9], a.c_fb = in[10], a.c_vxx = in[11], a.c_vx = in[12], a.c_fft = in[13], a.c_fbt = in[14];
  a.g_stage = out[0], a.g_term = out[1], a.g_G0 = out[2], a.g_g0 = out[3];
  r.mueq = mueq;
  r.mueq_b = mueq_b;
  run_instances(r.batch, nl, ab2::factor_adjoint_item_doubles(r.nx, r.nu, r.nc),
                [&](const EmuCtx &ctx, double *sm, long b) { ab2::factor_adjoint_item(a, ctx, sm, b); });
  return 0;
}

// bytes of shared memory one instance uses (nct, nc0, nth, chunk: not read)
extern "C" long emu_factor_adjoint_item_bytes(int nx, int nu, int nc, int nct, int nc0, int nth, int chunk) {
  return (long)ab2::factor_adjoint_item_doubles(nx, nu, nc) * (long)sizeof(double);
}
