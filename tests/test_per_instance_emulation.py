"""The sweep programs with a per-instance mu (ab2::InstanceMu, what the *_v launches run), executed on the CPU through
the host emulation (tests/emu_harness.py): the warp-per-instance group program with both step
implementations and both record-buffer layouts, the CTA-per-instance program, its leg mode and the stage-dense program.

Each instance's outputs must be array-equal to the scalar program run at that instance's mu; instances that share
their records but not their mu must differ where mu enters; and every instance matches the oracle at its own mu."""
import numpy as np
import pytest

import gen
from emu_harness import emulate
from oracle import gar_oracle as orc

MUS = (1.0, 1e-2, 1e-5)


def _batch(dims, seed):
    """Instances 0, 1, 2 share one problem (and get mu = 1, 1e-2, 1e-5); instance 3 is another problem."""
    nx, nu, nc, nct, N = dims
    a = gen.generate_batch(seed, 1, N, nx, nu, nc, nct)[0]
    b = gen.generate_batch(seed + 1, 1, N, nx, nu, nc, nct)[0]
    return [a, a.copy(), a.copy(), b], np.array([MUS[0], MUS[1], MUS[2], MUS[1]])


def _check(kind, dims, arg, legs=0, gains=True, seed=3):
    nx, nu, nc, nct, N = dims
    probs, mu_b = _batch(dims, seed + nx)
    # the group program with Vxx packed, as every device build runs it
    run = lambda mu: emulate(kind, probs, dims, mu, arg, packed=kind == "group", legs=legs)
    got = run(mu_b)
    want = {}
    for v in MUS:  # every instance as the scalar program at its own mu
        r = run(v)
        for k in r:
            if r[k].shape[0] == len(probs):  # (arrays of zero size are one-element placeholders)
                want.setdefault(k, np.empty_like(r[k]))[mu_b == v] = r[k][mu_b == v]
    for k in want:
        assert np.array_equal(got[k], want[k], equal_nan=True), (kind, k)
    assert np.all(got["status"] == 0)
    # the guard: same records, different mu -> different Z = C / mu, z = d / mu and multipliers
    for k in ("fbT", "ffT", "vsT") + (("vs",) if nc else ()):
        for i, j in ((0, 1), (1, 2), (0, 2)):
            assert not np.array_equal(got[k][i], got[k][j]), (kind, k, i, j)
    # each instance against the oracle at its own mu: the solution, and the feedback gains of the programs that compute
    # the proximal solver's (the legs' gains are parametric in the next leg's head, the dense program's are its own)
    stage, term, G0, g0 = gen.pack_problems(probs)
    for b in range(len(probs)):
        bo = orc.BatchedOracle(nx, nu, nc, nct, probs[0].nc0, N, 1, stage[b:b + 1], term[b:b + 1], G0[b:b + 1],
                               g0[b:b + 1])
        bo.sweep(mu_b[b], nthreads=1)
        ref = bo.get()
        for k in ("xs", "us", "vs", "lbdas"):
            if ref[k].size:
                assert gen.rel_fro(got[k][b], ref[k][0]) <= 1e-10, (kind, k, b, mu_b[b])
        if gains:
            assert gen.rel_fro(got["fb"][b, :, :nu], ref["fb"][0, :, :nu]) <= 1e-10, (kind, "K", b)


GROUP = [((2, 2, 2, 2, 6), m) for m in (0, 1)] + [((4, 2, 2, 2, 7), m) for m in (0, 1)] + \
    [((5, 2, 2, 2, 5), m) for m in (0, 1)] + [((12, 6, 6, 3, 4), m) for m in (0, 1)] + \
    [((12, 6, 0, 3, 5), m) for m in (2, 3)] + [((14, 7, 0, 2, 4), m) for m in (2, 3)]


@pytest.mark.parametrize("dims,mode", GROUP, ids=["%d_%d_%d_nct%d-mode%d" % (d[:4] + (m,)) for d, m in GROUP])
def test_group_program(dims, mode):
    """mode 0/1: lane-per-column step, single / double record buffer; 2/3: tensor-core step, double / single."""
    _check("group", dims, mode)


def test_cta_program_runtime_shape():
    _check("block", (7, 3, 2, 2, 6), 1)


def test_leg_mode():
    _check("legs", (4, 2, 2, 2, 8), 1, legs=3, gains=False)


def test_dense_program():
    _check("dense", (5, 3, 2, 2, 6), 1, gains=False)
