"""Leg mode of the CTA-per-instance program = gar::ParallelRiccatiSolver on the device
(gar/parallel-solver.hxx:51-243, gar/block-tridiagonal.hpp:52-182): the legs of every instance are
work items of ONE launch, the condensed block-tridiagonal system is solved by a second kernel, the
legs roll out in a third.  Host emulation (tests/emu_harness.py) against the oracle's restatement
of the parallel solver (same leg split) and against the serial solution."""
import numpy as np
import pytest

import gen
from emu_harness import emulate
from oracle import gar_oracle as orc


def oracle_parallel(prob, T, mueq):
    op = orc.OracleProblem(prob.copy())
    s = orc.ParallelRiccatiSolver(op, T, threaded=False)
    assert s.backward(mueq)
    sol = orc.OracleSolution(op)
    assert s.forward(sol)
    return op, s, sol


@pytest.mark.parametrize("shape", [(4, 2, 0, 0, 11, 2, 1e-8), (4, 2, 0, 0, 11, 3, 1e-8), (6, 3, 0, 0, 20, 4, 1e-8),
                                   (4, 2, 2, 0, 13, 2, 1e-3), (5, 3, 2, 2, 9, 3, 1e-2), (7, 3, 0, 0, 7, 8, 1e-8),
                                   (3, 2, 0, 0, 5, 6, 1e-8)])
def test_legs_match_oracle_parallel_and_serial(shape):
    nx, nu, nc, nct, N, T, mueq = shape
    B = 2
    probs = gen.generate_batch(40 + nx + T, B, N, nx, nu, nc, nct)
    got = emulate("legs", probs, (nx, nu, nc, nct, N), mueq, 1, legs=T)
    assert np.all(got["status"] == 0)
    cat = lambda v: np.concatenate([np.ravel(a) for a in v] + [np.zeros(0)])
    tol = 1e-10
    for b, p in enumerate(probs):
        op, s, sol = oracle_parallel(p, T, mueq)
        heads = [i * (N + 1) // T for i in range(T)]
        for t in range(N):
            f = s.factor(t)
            assert gen.rel_fro(got["fb"][b, t], f["fb"]) <= tol, ("fb", t)
            assert gen.rel_fro(got["ff"][b, t], f["ff"]) <= tol, ("ff", t)
            if f["dims"][4] > 0:
                assert gen.rel_fro(got["fth"][b, t], f["fth"]) <= tol, ("fth", t)
        for t in range(N + 1):
            f = s.factor(t)
            V = got["Vxx"][b, t].reshape(nx, nx).T
            assert gen.rel_fro(V, f["Vxx"]) <= tol, ("Vxx", t)
            if t in heads and t > 0:  # leg heads stay unsymmetrised, like datas[0] (SURVEY A1)
                pass
            assert gen.rel_fro(got["vx"][b, t], f["vx"]) <= tol
            if f["dims"][4] > 0:
                assert gen.rel_fro(got["Vxt"][b, t].reshape(nx, nx).T, f["Vxt"]) <= tol, ("Vxt", t)
                assert gen.rel_fro(got["Vtt"][b, t].reshape(nx, nx).T, f["Vtt"]) <= tol, ("Vtt", t)
                assert gen.rel_fro(got["vt"][b, t], f["vt"]) <= tol, ("vt", t)
        xs, us, vs, lb = sol.get()
        # the rollout: equal to the oracle's parallel solver (same algorithm) ...
        assert gen.rel_fro(got["xs"][b], np.stack(xs)) <= 1e-9
        assert gen.rel_fro(got["us"][b], np.stack(us[:N])) <= 1e-9
        assert gen.rel_fro(got["lbdas"][b], np.stack(lb[1:])) <= 1e-9
        assert gen.rel_fro(got["lbd0"][b], lb[0]) <= 1e-9
        if nc:
            assert gen.rel_fro(got["vs"][b], np.stack(vs[:N])) <= 1e-8
        # ... and to the serial solution at the reference's own thresholds (tests/gar/parallel.cpp:211-243)
        op2 = orc.OracleProblem(p)
        ser = orc.ProximalRiccatiSolver(op2)
        ser.backward(mueq)
        sol2 = orc.OracleSolution(op2)
        ser.forward(sol2)
        xs2, us2, vs2, lb2 = sol2.get()
        assert gen.rel_fro(got["xs"][b], np.stack(xs2)) <= 1e-7
        assert gen.rel_fro(got["us"][b], np.stack(us2[:N])) <= 1e-7
        assert gen.rel_fro(got["lbdas"][b], np.stack(lb2[1:])) <= 1e-7


def test_collapse_feedback_matches_the_reference_statement():
    """collapseFeedback (parallel-solver.hpp:41-51): K_0 -= Kth_0 * subdiagonal[1].  After the swap at
    parallel-solver.hxx:180-181 `subdiagonal[1]` is the ORIGINAL block Vxt_0^T, not the U factor the
    comment promises, so the result is not the serial solver's first gain; restated as written
    (oracle and device agree on it)."""
    nx, nu, N, T, mueq = 5, 2, 12, 3, 1e-8
    probs = gen.generate_batch(9, 1, N, nx, nu, 0, 0)
    got = emulate("legs", probs, (nx, nu, 0, 0, N), mueq, 1, legs=T, collapse=True)
    op, s, sol = oracle_parallel(probs[0], T, mueq)
    s.collapseFeedback()
    assert gen.rel_fro(got["fb"][0, 0, :nu], s.factor(0)["fb"][:nu]) <= 1e-10
