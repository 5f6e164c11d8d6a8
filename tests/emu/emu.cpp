// The host emulation library of the device programs: the warp-per-instance group program (group_emu.cpp), the
// CTA-per-instance program with its leg mode, and the stage-dense program (block_emu.cpp), and the per-item programs of
// resolve, the θ derivatives and the factorisation's derivatives (resolve_emu.cpp, theta_emu.cpp,
// factor_adjoint_emu.cpp, factor_tangent_emu.cpp), in one translation unit.
// TEST INFRASTRUCTURE.  Every entry point takes a complete ab2::SweepParams; the layout exports below let the
// caller's mirror of that struct check itself against this build.
#include <cstddef>
#include <cstring>

#include "../../aligator_b200/csrc/lq_record.cuh"
#include "block_emu.cpp"
#include "factor_adjoint_emu.cpp"
#include "factor_tangent_emu.cpp"
#include "group_emu.cpp"
#include "resolve_emu.cpp"
#include "theta_emu.cpp"

// Every shape `supported` (the library's ab2_gar_supported) accepts with nx, nu, nc < lim and nc0 in {0, 1, nx/2, nx},
// and with nct in {0, nx} and nth in {1, nx, 33} when `parametric` (nct = nth = 0 otherwise), for the item program
// whose item of one column or instance takes item_bytes(nx, nu, nc, nct, nc0, nth, 1) bytes of shared memory (one of
// the emu_*_item_bytes): how many are accepted (*accepted), how many of those need more than 227 KB (the return
// value; the first one in *bad = nx, nu, nc, nc0, nct, nth), and the largest item that fits, in bytes (*largest).
extern "C" long emu_item_size_scan(long (*item_bytes)(int, int, int, int, int, int, int), int parametric,
                                   int (*supported)(int, int, int, int), int lim, int *bad, long *largest,
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
          for (int t = 0; t < (parametric ? 2 : 1); ++t)
            for (int h = 0; h < (parametric ? 3 : 1); ++h) {
              const int nct = ncts[t], nth = parametric ? nths[h] : 0;
              ++*accepted;
              const long bytes = item_bytes(nx, nu, nc, nct, nc0, nth, 1);
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

extern "C" int emu_sweep_params_size() { return (int)sizeof(ab2::SweepParams); }

// offsetof(ab2::SweepParams, name), or -1 for a name that is not a field
extern "C" int emu_sweep_params_offset(const char *name) {
#define F(f) {#f, offsetof(ab2::SweepParams, f)},
  static const struct {
    const char *name;
    size_t off;
  } fields[] = {
      F(N) F(nct) F(nc0) F(batch) F(mueq) F(do_bwd) F(do_fwd)
      F(stage) F(term) F(G0) F(g0)
      F(ff) F(fb) F(Vxx) F(vx) F(ffT) F(fbT) F(kkt0)
      F(xs) F(us) F(vs) F(vsT) F(lbd0) F(lbdas) F(status) F(pivstat)
      F(stagger_ns) F(num_sms) F(ctas_per_sm) F(stage_head)
      F(nth) F(theta) F(fth) F(Vxt) F(Vtt) F(vt) F(kkt0fth) F(thGrad) F(thHess)
      F(legs) F(clk) F(cond)
      F(peer_world) F(peer_dst) F(peer_off)
      F(Vxx0) F(mueq_b)
  };
#undef F
  for (const auto &f : fields)
    if (std::strcmp(f.name, name) == 0)
      return (int)f.off;
  return -1;
}

// the record layouts of lq_record.cuh, for the tests' mirror of them.  Stage: A B f Q S R q r C D d end, the tail
// Gx Gu Gv Gth gamma end, the stored length and the triangle-packed length (20 ints).  Terminal: Q q C d end, the tail
// Gx Gv Gth gamma end and the length (11 ints).
extern "C" void emu_stage_layout(int nx, int nu, int nc, int nth, int *out) {
  const ab2::StageOffsets o = ab2::stage_offsets(nx, nu, nc);
  const ab2::TailOffsets t = ab2::stage_tail(o, nx, nu, nc, nth);
  const int v[] = {o.A, o.B, o.f, o.Q, o.S, o.R, o.q, o.r, o.C, o.D, o.d, o.end, t.Gx, t.Gu, t.Gv, t.Gth, t.gamma, t.end,
                   ab2::stage_record_len(nx, nu, nc, nth), ab2::stage_sym_len(nx, nu, nc)};
  std::memcpy(out, v, sizeof(v));
}
extern "C" void emu_term_layout(int nx, int nct, int nth, int *out) {
  const ab2::TermOffsets o = ab2::term_offsets(nx, nct);
  const ab2::TailOffsets t = ab2::term_tail(o, nx, nct, nth);
  const int v[] = {o.Q, o.q, o.C, o.d, o.end, t.Gx, t.Gv, t.Gth, t.gamma, t.end, ab2::term_record_len(nx, nct, nth)};
  std::memcpy(out, v, sizeof(v));
}
