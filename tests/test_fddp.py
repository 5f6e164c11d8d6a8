"""SolverFDDP::backwardPass (solvers/fddp/solver-fddp.hxx:204-277): the numpy restatement against the
recursion's defining equations (CPU), and ab2_fddp_backward_pass on the device against the restatement (GPU)."""
import numpy as np
import pytest

import gen
from inner_cases import random_fddp
from oracle import fddp as of


def test_restatement_satisfies_the_recursion():
    rng = np.random.default_rng(0)
    B, N, nx, nu, preg = 1, 6, 4, 2, 1e-3
    d = random_fddp(rng, B, N, nx, nu)
    r = of.backward_pass(*[list(d[k][0]) for k in ("Jx", "Ju")], list(d["fs"][0]), *[list(d[k][0]) for k in
                         ("Lxx", "Lxu", "Luu", "Lx", "Lu")], d["Lxx_N"][0], d["Lx_N"][0], preg)
    for i in range(N):  # Quu k = -Qu and Quu K = -Qux (the LLT solve), Quuks = Quu k
        J = np.hstack([d["Jx"][0, i], d["Ju"][0, i]])
        hess = np.block([[d["Lxx"][0, i], d["Lxu"][0, i]], [d["Lxu"][0, i].T, d["Luu"][0, i]]]) + J.T @ r["Vxx"][i + 1] @ J
        grad = np.concatenate([d["Lx"][0, i], d["Lu"][0, i]]) + J.T @ r["Vx"][i + 1]
        Quu = hess[nx:, nx:] + preg * np.eye(nu)
        assert np.allclose(Quu @ r["k"][i], -grad[nx:], atol=1e-12)
        assert np.allclose(Quu @ r["K"][i], -hess[nx:, :nx], atol=1e-12)
        assert np.allclose(r["Quuks"][i], -grad[nx:], atol=1e-12)
        assert np.array_equal(r["Vxx"][i], r["Vxx"][i].T)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(12, 6, 30, 9), (6, 3, 20, 5), (14, 7, 25, 4), (9, 4, 10, 3)])
def test_device_fddp_backward_pass(shape):
    import torch
    assert torch.cuda.is_available()
    import __graft_entry__ as g
    g.build()
    import aligator_b200.gar as gar
    nx, nu, N, B = shape
    preg = 1e-4
    rng = np.random.default_rng(nx)
    d = random_fddp(rng, B, N, nx, nu)
    dev = torch.device("cuda:0")
    cm = lambda a: np.ascontiguousarray(np.swapaxes(a, -1, -2))  # column-major blocks
    arr = {k: torch.tensor(cm(d[k]) if d[k].ndim >= 3 and k not in ("fs", "Lx", "Lu", "Lx_N") else d[k], device=dev)
           for k in d}
    s = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B)
    Vx = torch.empty(B, N + 1, nx, dtype=torch.float64, device=dev)
    Qk = torch.empty(B, N, nu, dtype=torch.float64, device=dev)
    s.fddp_backward_pass(arr, preg, Vx, Qk)
    s.synchronize()
    assert np.all(s.status() == 0)
    fb, ff, V = s.get(gar.OUT_FB), s.get(gar.OUT_FF), s.get(gar.OUT_VXX)
    Vx, Qk = Vx.cpu().numpy(), Qk.cpu().numpy()
    il = np.tril_indices(nx)
    for b in range(B):
        r = of.backward_pass(list(d["Jx"][b]), list(d["Ju"][b]), list(d["fs"][b]), list(d["Lxx"][b]), list(d["Lxu"][b]),
                             list(d["Luu"][b]), list(d["Lx"][b]), list(d["Lu"][b]), d["Lxx_N"][b], d["Lx_N"][b], preg)
        for i in range(N):
            assert gen.rel_fro(fb[b, i, :nu], r["K"][i]) <= 1e-10
            assert gen.rel_fro(ff[b, i, :nu], r["k"][i]) <= 1e-10
            assert gen.rel_fro(Qk[b, i], r["Quuks"][i]) <= 1e-10
        for i in range(N + 1):
            assert gen.rel_fro(V[b, i][il], r["Vxx"][i][il]) <= 1e-10
            assert gen.rel_fro(Vx[b, i], r["Vx"][i]) <= 1e-10
    s.close()
