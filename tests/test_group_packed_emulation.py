"""The group program with Vxx stored as packed lower triangles (vxx_layout.h, the layout every device
build uses) against the full-layout program it replaced, both executed on the CPU through the host
emulation: after expansion every output must be bit-identical."""
import numpy as np
import pytest

import gen
from emu_harness import emulate, lib


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
    probs = gen.generate_batch(11 + nx + N, 2, N, nx, nu, nc, nct)
    ref = emulate("group", probs, (nx, nu, nc, nct, N), mueq, mode, packed=False)
    got = emulate("group", probs, (nx, nu, nc, nct, N), mueq, mode, packed=True)
    assert np.all(ref["status"] == 0)
    P = lib().emu_vxx_packed_doubles(nx)
    assert P % 2 == 0 and P - nx * (nx + 1) // 2 in (0, 1)
    if N > 0 and P > nx * (nx + 1) // 2:
        assert np.all(got["Vxx"][:, 1:, P - 1] == 0.0)  # the padding entry is written
    got["Vxx"] = expand(got, nx, N)
    for k in ("ff", "fb", "Vxx", "vx", "ffT", "fbT", "kkt0", "xs", "us", "vs", "vsT", "lbd0", "lbdas", "status",
              "pivstat"):
        assert np.array_equal(got[k], ref[k], equal_nan=True), k
