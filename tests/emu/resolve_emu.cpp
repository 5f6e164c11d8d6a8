// Host emulation of the ab2_gar_resolve program (aligator_b200/csrc/lq_resolve.cuh): each work item runs on `nl`
// emulated lanes (item_emu.h).  Part of the emulation library (emu.cpp).
#include "../../aligator_b200/csrc/lq_resolve.cuh"
#include "item_emu.h"

// dims: batch, N, nx, nu, nc, nct, nc0, srec, trec, stage_head, nrhs, chunk, lanes
// in:   stage, term, G0, fb, fbT, Vxx, Vxx0, q, r, d, dN, g0, f     out: xs, us, vs, vsT, lam0, lams
extern "C" int emu_resolve(const int *dims, double mueq, const double *mueq_b, const double *const *in,
                           double *const *out) {
  ab2::ResolveArgs a{};
  a.batch = dims[0], a.N = dims[1], a.nx = dims[2], a.nu = dims[3], a.nc = dims[4], a.nct = dims[5], a.nc0 = dims[6];
  a.srec = dims[7], a.trec = dims[8], a.stage_head = dims[9], a.nrhs = dims[10], a.chunk = dims[11];
  const int nl = dims[12];
  a.stage = in[0], a.term = in[1], a.G0 = in[2], a.fb = in[3], a.fbT = in[4], a.Vxx = in[5], a.Vxx0 = in[6];
  a.q = in[7], a.r = in[8], a.d = in[9], a.dN = in[10], a.g0 = in[11], a.f = in[12];
  a.xs = out[0], a.us = out[1], a.vs = out[2], a.vsT = out[3], a.lam0 = out[4], a.lams = out[5];
  a.mueq = mueq;
  a.mueq_b = mueq_b;
  run_chunks(a.batch, a.nrhs, a.chunk, nl, ab2::resolve_item_doubles(a.nx, a.nu, a.nc, a.nc0, a.chunk),
             [&](const EmuCtx &ctx, double *sm, long b, int j0, int R) { ab2::resolve_item(a, ctx, sm, b, j0, R); });
  return 0;
}

// bytes of shared memory one item of `chunk` right-hand sides uses (nct, nth: not read)
extern "C" long emu_resolve_item_bytes(int nx, int nu, int nc, int nct, int nc0, int nth, int chunk) {
  return (long)ab2::resolve_item_doubles(nx, nu, nc, nc0, chunk) * (long)sizeof(double);
}
