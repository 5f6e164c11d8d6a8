"""The group program with Vxx stored as packed lower triangles (vxx_layout.h, the layout every device
build uses) against the full-layout program it replaced, both executed on the CPU through the host
emulation: after expansion every output must be bit-identical."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import gen
from test_group_emulation import SweepParams, _dp

HERE = os.path.dirname(os.path.abspath(__file__))
EMU_DIR = os.path.join(HERE, "emu")
EMU_LIB = os.path.join(EMU_DIR, "libgroup_packed_emu.so")
CSRC = os.path.join(HERE, "..", "aligator_b200", "csrc")


class SweepParamsPacked(C.Structure):
    _fields_ = SweepParams._fields_ + [("Vxx0", _dp)]


def _lib():
    srcs = [os.path.join(EMU_DIR, "group_packed_emu.cpp"), os.path.join(EMU_DIR, "group_emu.cpp")] + \
        [os.path.join(CSRC, f) for f in ("riccati_group.cuh", "riccati_configs.h", "vxx_layout.h")]
    if (not os.path.exists(EMU_LIB)
            or os.path.getmtime(EMU_LIB) < max(os.path.getmtime(s) for s in srcs)):
        subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++20", "-fPIC", "-shared", "-pthread",
                               "-o", EMU_LIB, srcs[0]])
    return C.CDLL(EMU_LIB)


def run(lib, nx, nu, nc, nct, N, probs, mueq, mode, packed):
    B, nc0 = len(probs), probs[0].nc0
    stage, term, G0, g0 = gen.pack_problems(probs)
    srec = lib.emu_stage_record(nx, nu, nc)
    if N > 0 and stage.shape[-1] != srec:
        stage = np.concatenate([stage, np.zeros(stage.shape[:-1] + (srec - stage.shape[-1],))], -1)
    stage = np.ascontiguousarray(stage)
    nr, P = nu + nc + nx, lib.emu_vxx_packed_doubles(nx)
    z = lambda *s: np.full(s if np.prod(s) > 0 else (1,), np.nan)
    out = dict(ff=z(B, N, nr), fb=z(B, N, nr, nx), Vxx=z(B, N + 1, P if packed else nx * nx), vx=z(B, N + 1, nx),
               ffT=z(B, nct), fbT=z(B, nct, nx), kkt0=z(B, nx + nc0), xs=z(B, N + 1, nx),
               us=z(B, N, nu), vs=z(B, N, nc), vsT=z(B, nct), lbd0=z(B, nc0), lbdas=z(B, N, nx))
    if packed:
        out["Vxx0"] = z(B, nx * nx)
    status, pivstat = np.full(B, -1, dtype=np.int32), np.zeros(B, dtype=np.int32)
    p = SweepParamsPacked() if packed else SweepParams()
    p.N, p.nct, p.nc0, p.batch, p.mueq, p.do_bwd, p.do_fwd = N, nct, nc0, B, mueq, 1, 1
    for k, v in dict(stage=stage, term=term, G0=G0, g0=g0, **out).items():
        setattr(p, k, v.ctypes.data_as(_dp))
    p.status = status.ctypes.data_as(C.POINTER(C.c_int))
    p.pivstat = pivstat.ctypes.data_as(C.POINTER(C.c_int))
    rc = (lib.emu_sweep_packed if packed else lib.emu_sweep)(nx, nu, nc, mode, C.byref(p))
    assert rc == 0
    out["status"], out["pivstat"] = status, pivstat
    return out


def expand(out, nx, N):
    """[B][N+1][nx*nx] column-major blocks from the packed layout: slot 0 from the full array."""
    pk, B = out["Vxx"], out["Vxx"].shape[0]
    full = np.empty((B, N + 1, nx * nx))
    full[:, 0] = out["Vxx0"]
    for t in range(1, N + 1):
        for j in range(nx):
            for i in range(nx):
                a, b = max(i, j), min(i, j)
                full[:, t, i + j * nx] = pk[:, t, b * nx - b * (b - 1) // 2 + (a - b)]
    return full


SHAPES = [(2, 2, 0, 8), (2, 2, 2, 8), (3, 2, 0, 8), (4, 2, 2, 8), (4, 2, 0, 8), (5, 2, 2, 16), (6, 3, 0, 16),
          (8, 3, 0, 16), (10, 4, 0, 32), (12, 6, 0, 32), (12, 6, 6, 32), (14, 7, 0, 32)]
CASES = [(s, m) for s in SHAPES for m in (0, 1, 2, 3) if m < 2 or (s[3] == 32 and s[2] == 0 and s[0] % 2 == 0)]


@pytest.mark.parametrize("N", [0, 1, 2, 7])
@pytest.mark.parametrize("shape,mode", CASES)
def test_packed_vxx_program_is_bit_identical(shape, mode, N):
    """mode 0/1: lane-per-column step, single/double record buffer; 2/3: tensor-core step, double/single."""
    nx, nu, nc, _ = shape
    nct = 2 if N == 2 else 0
    mueq = 1e-3 if (nc or nct) else 1e-8
    lib = _lib()
    probs = gen.generate_batch(11 + nx + N, 2, N, nx, nu, nc, nct)
    ref = run(lib, nx, nu, nc, nct, N, probs, mueq, mode, packed=False)
    got = run(lib, nx, nu, nc, nct, N, probs, mueq, mode, packed=True)
    assert np.all(ref["status"] == 0)
    P = lib.emu_vxx_packed_doubles(nx)
    assert P % 2 == 0 and P - nx * (nx + 1) // 2 in (0, 1)
    if N > 0 and P > nx * (nx + 1) // 2:
        assert np.all(got["Vxx"][:, 1:, P - 1] == 0.0)  # the padding entry is written
    got["Vxx"] = expand(got, nx, N)
    for k in ("ff", "fb", "Vxx", "vx", "ffT", "fbT", "kkt0", "xs", "us", "vs", "vsT", "lbd0", "lbdas", "status",
              "pivstat"):
        assert np.array_equal(got[k], ref[k], equal_nan=True), k
