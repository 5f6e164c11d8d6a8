// The host emulation library of the device programs: the warp-per-instance group program (group_emu.cpp), the
// CTA-per-instance program with its leg mode, and the stage-dense program (block_emu.cpp), and the per-item programs of
// resolve and the factorisation's derivatives (resolve_emu.cpp, factor_adjoint_emu.cpp, factor_tangent_emu.cpp), in one
// translation unit.
// TEST INFRASTRUCTURE.  Every entry point takes a complete ab2::SweepParams; the layout exports below let the
// caller's mirror of that struct check itself against this build.
#include <cstddef>
#include <cstring>

#include "block_emu.cpp"
#include "factor_adjoint_emu.cpp"
#include "factor_tangent_emu.cpp"
#include "group_emu.cpp"
#include "resolve_emu.cpp"

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
