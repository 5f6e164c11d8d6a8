// Host emulation of the group program with Vxx stored packed (Cfg::VXX_PACKED, vxx_layout.h), beside the
// full-layout program of group_emu.cpp, which stays the reference it is compared with.  TEST INFRASTRUCTURE.
#include "group_emu.cpp"

template <int NX, int NU, int NC, int G> int dispatch_packed(int mode, const ab2::SweepParams &p) {
  if (mode >= 2) { // tensor-core formulation (3: single record buffer)
    if constexpr (G == 32 && NC == 0 && NX % 2 == 0)
      return mode == 2 ? run<ab2::Cfg<NX, NU, NC, G, true, true, true, true>>(p)
                       : run<ab2::Cfg<NX, NU, NC, G, false, true, true, true>>(p);
    else
      return 3;
  }
  return mode ? run<ab2::Cfg<NX, NU, NC, G, true, true, false, true>>(p)
              : run<ab2::Cfg<NX, NU, NC, G, false, true, false, true>>(p);
}

extern "C" int emu_vxx_packed_doubles(int nx) { return ab2::vxx_packed_doubles(nx); }

extern "C" int emu_sweep_packed(int nx, int nu, int nc, int db, const ab2::SweepParams *p) {
#define X(NX, NU, NC, G)                                                        \
  if (nx == NX && nu == NU && nc == NC)                                         \
    return dispatch_packed<NX, NU, NC, G>(db, *p);
  AB2_FOR_EACH_CONFIG(X)
#undef X
  return 1;
}
