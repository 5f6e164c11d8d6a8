"""The stage-dense solver on the device (aligator_b200/csrc/riccati_dense.cuh = gar::RiccatiSolverDense): host
emulation against the oracle's restatement of the same algorithm and against the proximal solution."""
import numpy as np
import pytest

import gen
from aligator_b200.lqr import LqrKnot
from emu_harness import emulate
from oracle import gar_oracle as orc


@pytest.mark.parametrize("shape", [(4, 2, 0, 0, 8, 1e-8, 1), (6, 3, 0, 0, 12, 1e-8, 1), (4, 2, 2, 0, 9, 1e-3, 1),
                                   (5, 3, 2, 2, 7, 1e-2, 1), (12, 6, 0, 0, 6, 1e-8, 1), (14, 7, 3, 0, 4, 1e-3, 2)])
def test_dense_kernel_matches_oracle_dense_and_proximal(shape):
    nx, nu, nc, nct, N, mueq, nw = shape
    probs = gen.generate_batch(50 + nx, 2, N, nx, nu, nc, nct)
    got = emulate("dense", probs, (nx, nu, nc, nct, N), mueq, nw)
    assert np.all(got["status"] == 0)
    n = nu + nc + 2 * nx
    for b, p in enumerate(probs):
        q = p.copy()
        kt = q.stages[-1]
        k0 = LqrKnot(nx, 0, nct, 0)  # the dense solver's terminal knot (nx2 = 0), see tests/test_oracle_dense.py
        k0.Q[:], k0.q[:], k0.C[:], k0.d[:] = kt.Q, kt.q, kt.C, kt.d
        q.stages[-1] = k0
        op = orc.OracleProblem(q)
        dn = orc.RiccatiSolverDense(op)
        assert dn.backward(mueq)
        sol = orc.OracleSolution(op)
        dn.forward(sol)
        for t in range(N):
            f = dn.factor(t)
            assert gen.rel_fro(got["fb"][b, t], f["fb"]) <= 1e-10, ("fb", t)
            assert gen.rel_fro(got["ff"][b, t], f["ff"]) <= 1e-10, ("ff", t)
        for t in range(N + 1):
            f = dn.factor(t)
            assert gen.rel_fro(got["Vxx"][b, t].reshape(nx, nx).T, f["Pxx"]) <= 1e-10
            assert gen.rel_fro(got["vx"][b, t], f["px"]) <= 1e-10
        xs, us, vs, lb = sol.get()
        assert gen.rel_fro(got["xs"][b], np.stack(xs)) <= 1e-10 and gen.rel_fro(got["us"][b], np.stack(us)) <= 1e-10
        assert gen.rel_fro(got["lbdas"][b], np.stack(lb[1:])) <= 1e-10
        # and the proximal algorithm's solution of the same problem
        op2 = orc.OracleProblem(p)
        pr = orc.ProximalRiccatiSolver(op2)
        pr.backward(mueq)
        s2 = orc.OracleSolution(op2)
        pr.forward(s2)
        xs2, us2, _, lb2 = s2.get()
        assert gen.rel_fro(got["xs"][b], np.stack(xs2)) <= 1e-9 and gen.rel_fro(got["us"][b], np.stack(us2[:N])) <= 1e-9
