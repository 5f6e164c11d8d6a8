"""The emulation helper's ctypes mirror of ab2::SweepParams against the struct the library was compiled with."""
from emu_harness import SweepParams, layout_mismatches, lib


def test_sweep_params_mirror_matches_the_library():
    """Same size and the same offset for every field: a mirror that ends early would let the library read past the
    caller's buffer."""
    assert not layout_mismatches(lib(), SweepParams)
