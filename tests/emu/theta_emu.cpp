// Host emulation of the ab2_gar_theta_tangent and ab2_gar_theta_adjoint programs (aligator_b200/csrc/lq_theta.cuh):
// each work item runs on `nl` emulated lanes (item_emu.h).  Built as a library of its own (tests/theta_emu_harness.py).
#include "../../aligator_b200/csrc/lq_theta.cuh"
#include "item_emu.h"

#include <vector>

// dims: batch, N, nx, nu, nc, nct, nc0, nth, nrhs, chunk, lanes, adjoint (0: tangent, 1: adjoint)
// in:   fb, fth, fbT, Vxx, Vxt, kkt0fth, then dtheta (tangent) or cxs, cus, cvs, cvsT, clam0, clams (adjoint)
// out:  xs, us, vs, vsT, lam0, lams (tangent) or theta_bar (adjoint)
extern "C" int emu_theta(const int *dims, const double *const *in, double *const *out) {
  ab2::ThetaArgs a{};
  a.batch = dims[0], a.N = dims[1], a.nx = dims[2], a.nu = dims[3], a.nc = dims[4], a.nct = dims[5], a.nc0 = dims[6];
  a.nth = dims[7], a.nrhs = dims[8], a.chunk = dims[9];
  const int nl = dims[10];
  const bool adjoint = dims[11] != 0;
  a.fb = in[0], a.fth = in[1], a.fbT = in[2], a.Vxx = in[3], a.Vxt = in[4], a.kkt0fth = in[5];
  if (adjoint) {
    a.cxs = in[6], a.cus = in[7], a.cvs = in[8], a.cvsT = in[9], a.clam0 = in[10], a.clams = in[11];
    a.theta_bar = out[0];
  } else {
    a.dtheta = in[6];
    a.xs = out[0], a.us = out[1], a.vs = out[2], a.vsT = out[3], a.lam0 = out[4], a.lams = out[5];
  }
  const int chunks = (a.nrhs + a.chunk - 1) / a.chunk;
  std::vector<double> sm(ab2::theta_item_doubles(a.nx, a.nu, a.nc, a.nct, a.nc0, a.nth, a.chunk));
  for (long b = 0; b < a.batch; ++b)
    for (int c = 0; c < chunks; ++c) {
      const int j0 = c * a.chunk, R = a.nrhs - j0 < a.chunk ? a.nrhs - j0 : a.chunk;
      run_lanes(nl, [&](const EmuCtx &ctx) {
        if (adjoint)
          ab2::theta_adjoint_item(a, ctx, sm.data(), b, j0, R);
        else
          ab2::theta_tangent_item(a, ctx, sm.data(), b, j0, R);
      });
    }
  return 0;
}

// bytes of shared memory one item of `chunk` directions uses
extern "C" long emu_theta_item_bytes(int nx, int nu, int nc, int nct, int nc0, int nth, int chunk) {
  return (long)ab2::theta_item_doubles(nx, nu, nc, nct, nc0, nth, chunk) * (long)sizeof(double);
}

// Every shape `supported` (the library's ab2_gar_supported) accepts with nx, nu, nc < lim, nc0 in {0, 1, nx/2, nx},
// nct in {0, nx} and nth in {1, nx, 33}: how many are accepted (*accepted), how many of those need more than 227 KB of
// shared memory for one direction (the return value; the first one in *bad = nx, nu, nc, nc0, nct, nth), and the
// largest item that fits, in bytes (*largest).
extern "C" long emu_theta_size_scan(int (*supported)(int, int, int, int), int lim, int *bad, long *largest,
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
          const int ncts[2] = {0, nx}, nths[3] = {1, nx, 33};
          for (int nct : ncts)
            for (int nth : nths) {
              ++*accepted;
              const long bytes = emu_theta_item_bytes(nx, nu, nc, nct, nc0, nth, 1);
              if (bytes > 227 * 1024) {
                if (over++ == 0)
                  bad[0] = nx, bad[1] = nu, bad[2] = nc, bad[3] = nc0, bad[4] = nct, bad[5] = nth;
              } else if (bytes > *largest) {
                *largest = bytes;
              }
            }
        }
      }
  return over;
}
