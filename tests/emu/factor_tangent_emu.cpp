// Host emulation of the ab2_gar_factor_tangent program (aligator_b200/csrc/lq_factor_tangent.cuh): each instance runs
// on `nl` emulated lanes (item_emu.h).  Part of the emulation library (emu.cpp).
#include "../../aligator_b200/csrc/lq_factor_tangent.cuh"
#include "item_emu.h"

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
  run_instances(r.batch, nl, ab2::factor_tangent_item_doubles(r.nx, r.nu, r.nc),
                [&](const EmuCtx &ctx, double *sm, long b) { ab2::factor_tangent_item(a, ctx, sm, b); });
  return 0;
}

// bytes of shared memory one instance uses (nct, nc0, nth, chunk: not read)
extern "C" long emu_factor_tangent_item_bytes(int nx, int nu, int nc, int nct, int nc0, int nth, int chunk) {
  return (long)ab2::factor_tangent_item_doubles(nx, nu, nc) * (long)sizeof(double);
}
