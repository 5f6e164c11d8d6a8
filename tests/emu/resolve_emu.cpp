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
  const int chunks = (a.nrhs + a.chunk - 1) / a.chunk;
  std::vector<double> sm(ab2::resolve_item_doubles(a.nx, a.nu, a.nc, a.nc0, a.chunk));
  for (long b = 0; b < a.batch; ++b)
    for (int c = 0; c < chunks; ++c) {
      const int j0 = c * a.chunk, R = a.nrhs - j0 < a.chunk ? a.nrhs - j0 : a.chunk;
      run_lanes(nl, [&](const EmuCtx &ctx) { ab2::resolve_item(a, ctx, sm.data(), b, j0, R); });
    }
  return 0;
}

// Every shape `supported` (the library's ab2_gar_supported) accepts with nx, nu, nc < lim and nc0 in {0, 1, nx/2, nx}:
// how many need more than 227 KB of shared memory for one right-hand side (the first one in *bad = nx, nu, nc, nc0),
// and the largest item in bytes (*largest).
extern "C" long emu_resolve_size_scan(int (*supported)(int, int, int, int), int lim, int *bad, long *largest) {
  long over = 0;
  *largest = 0;
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
          const long bytes = (long)ab2::resolve_item_doubles(nx, nu, nc, nc0, 1) * (long)sizeof(double);
          *largest = bytes > *largest ? bytes : *largest;
          if (bytes > 227 * 1024 && over++ == 0)
            bad[0] = nx, bad[1] = nu, bad[2] = nc, bad[3] = nc0;
        }
      }
  return over;
}
