"""Parametric problems (nth > 0: riccati-kernel.hxx:185-192, 278-311; proximal-riccati.hxx:50-59;
forward with theta) on the CTA-per-instance program, host emulation vs the oracle."""
import numpy as np
import pytest

import gen
from emu_harness import emulate
from lq_cases import make_problem
from oracle import gar_oracle as orc


# (nx, nu, nc, nct, nth, N, mueq, warps[, Gv != 0])
@pytest.mark.parametrize("shape", [(5, 2, 0, 0, 3, 6, 1e-8, 1), (4, 3, 2, 0, 2, 5, 1e-3, 1), (7, 3, 0, 2, 7, 4, 1e-2, 2),
                                   (6, 2, 1, 0, 1, 3, 1e-3, 1), (4, 3, 2, 0, 2, 5, 1e-3, 1, True),
                                   (5, 2, 2, 2, 3, 4, 1e-2, 1, True)])
def test_parametric_block_sweep(shape):
    nx, nu, nc, nct, nth, N, mueq, nw = shape[:8]
    p = make_problem(sum(shape[:6]), N, nx, nu, nc, nct, nth, gv=len(shape) > 8 and shape[8])
    theta = np.random.default_rng(3).standard_normal(nth)
    got = emulate("parametric", [p], (nx, nu, nc, nct, N), mueq, nw, nth=nth, theta=theta)
    assert got["status"][0] == 0
    op = orc.OracleProblem(p)
    ref = orc.ProximalRiccatiSolver(op)
    assert ref.backward(mueq)
    tol = 1e-9 if (nc or nct) else 1e-10
    for t in range(N):
        f = ref.factor(t)
        for key, a, b in (("fb", got["fb"][0, t], f["fb"]), ("ff", got["ff"][0, t], f["ff"]),
                          ("fth", got["fth"][0, t], f["fth"])):
            assert gen.rel_fro(a, b) <= tol, (t, key)
    for t in range(N + 1):
        f = ref.factor(t)
        assert gen.rel_fro(got["Vxt"][0, t].reshape(nth, nx).T, f["Vxt"]) <= tol, t
        assert gen.rel_fro(got["Vtt"][0, t].reshape(nth, nth).T, f["Vtt"]) <= tol, t
        assert gen.rel_fro(got["vt"][0, t], f["vt"]) <= tol, t
    k0 = ref.kkt0()
    assert gen.rel_fro(got["kkt0"][0], k0["ff"]) <= tol
    assert gen.rel_fro(got["kkt0fth"][0], k0["fth"]) <= tol
    assert gen.rel_fro(got["thGrad"][0], k0["thGrad"]) <= tol
    assert gen.rel_fro(got["thHess"][0].reshape(nth, nth).T, k0["thHess"]) <= tol
    sol = orc.OracleSolution(op)
    assert ref.forward(sol, theta)
    xs, us, vs, lb = sol.get()
    assert gen.rel_fro(got["xs"][0], np.array(xs)) <= tol
    assert gen.rel_fro(got["us"][0], np.array(us[:N])) <= tol
    assert gen.rel_fro(got["lbd0"][0], lb[0]) <= tol
    assert gen.rel_fro(got["lbdas"][0], np.array(lb[1:])) <= tol


def test_parametric_random_shapes():
    """Seeded random sweep: odd sizes, constrained / terminal-constrained, nth from 1 to nx."""
    rng = np.random.default_rng(99)
    done = 0
    while done < 10:
        nx, nu = int(rng.integers(1, 9)), int(rng.integers(1, 5))
        nc = int(rng.integers(0, 3)) if rng.random() < 0.4 else 0
        nct = int(rng.integers(0, 3)) if rng.random() < 0.3 else 0
        nth = int(rng.integers(1, nx + 1))
        N = int(rng.integers(0, 5))
        need = max(nx + 1, nu + nc, 2 * nx, nu + nc + nx, nth)
        nw = (need + 31) // 32
        mueq = 1e-3 if (nc or nct) else 1e-8
        test_parametric_block_sweep((nx, nu, nc, nct, nth, N, mueq, nw))
        done += 1
