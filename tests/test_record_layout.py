"""The tests' mirror of the knot-record layouts (lq_adjoint_ref.stage_offsets / term_offsets) against the one
definition in csrc/lq_record.cuh, as exported by the emulation library: every compile-time shape of
riccati_configs.h, config 5, constrained and parametric records, nu = 0 and nx = 1."""
import ctypes as C

import numpy as np
import pytest

import emu_harness
import lq_adjoint_ref as ref
from aligator_b200 import build

STAGE = ("A", "B", "f", "Q", "S", "R", "q", "r", "C", "D", "d")
TAIL = ("Gx", "Gu", "Gv", "Gth", "gamma")
TERM = ("Q", "q", "C", "d")
TERM_TAIL = ("Gx", "Gv", "Gth", "gamma")
SHAPES = sorted({(nx, nu, nc) for (nx, nu, nc, _) in build.configs()}
                | {(57, 28, 0), (56, 22, 0), (4, 2, 2), (4, 2, 1), (6, 3, 5), (5, 0, 0), (5, 0, 2), (1, 1, 0), (1, 3, 2)})


def _starts(off, names, length):
    return [off[k][0] for k in names] + [length]


@pytest.mark.parametrize("nth", [0, 1, 3])
@pytest.mark.parametrize("nx,nu,nc", SHAPES)
def test_stage_layout_matches_header(nx, nu, nc, nth):
    out = np.zeros(20, dtype=np.int32)
    emu_harness.lib().emu_stage_layout(nx, nu, nc, nth, out.ctypes.data_as(C.POINTER(C.c_int)))
    plain, _ = ref.stage_offsets(nx, nu, nc)
    off, srec = ref.stage_offsets(nx, nu, nc, nth)
    end = plain["d"][1]
    assert list(out[:12]) == _starts(plain, STAGE, end)
    tail = _starts(off, TAIL, off["gamma"][1]) if nth else [end] * 6
    assert list(out[12:18]) == tail
    assert out[18] == srec and srec % 2 == 0
    assert out[19] == end - nx * (nx - 1) // 2 - nu * (nu - 1) // 2  # lower triangles of Q and R


@pytest.mark.parametrize("nth", [0, 1, 3])
@pytest.mark.parametrize("nx,nct", [(1, 0), (4, 2), (12, 0), (57, 0), (6, 5)])
def test_term_layout_matches_header(nx, nct, nth):
    out = np.zeros(11, dtype=np.int32)
    emu_harness.lib().emu_term_layout(nx, nct, nth, out.ctypes.data_as(C.POINTER(C.c_int)))
    plain, _ = ref.term_offsets(nx, nct)
    off, trec = ref.term_offsets(nx, nct, nth)
    end = plain["d"][1]
    assert list(out[:5]) == _starts(plain, TERM, end)
    assert list(out[5:10]) == (_starts(off, TERM_TAIL, off["gamma"][1]) if nth else [end] * 5)
    assert out[10] == trec
