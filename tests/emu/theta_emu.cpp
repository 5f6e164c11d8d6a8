// Host emulation of the ab2_gar_theta_tangent and ab2_gar_theta_adjoint programs (aligator_b200/csrc/lq_theta.cuh):
// each work item runs on `nl` emulated lanes (item_emu.h).  Part of the emulation library (emu.cpp).
#include "../../aligator_b200/csrc/lq_theta.cuh"
#include "item_emu.h"

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
  run_chunks(a.batch, a.nrhs, a.chunk, nl, ab2::theta_item_doubles(a.nx, a.nu, a.nc, a.nct, a.nc0, a.nth, a.chunk),
             [&](const EmuCtx &ctx, double *sm, long b, int j0, int R) {
               if (adjoint)
                 ab2::theta_adjoint_item(a, ctx, sm, b, j0, R);
               else
                 ab2::theta_tangent_item(a, ctx, sm, b, j0, R);
             });
  return 0;
}

// bytes of shared memory one item of `chunk` directions uses
extern "C" long emu_theta_item_bytes(int nx, int nu, int nc, int nct, int nc0, int nth, int chunk) {
  return (long)ab2::theta_item_doubles(nx, nu, nc, nct, nc0, nth, chunk) * (long)sizeof(double);
}
