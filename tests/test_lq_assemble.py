"""LQ assembly (updateLQSubproblem + computeProjectedJacobians, solver-proxddp.hxx:25-69,
734-805): the numpy oracle against a hand-computed case (CPU) and the CUDA kernel against the
oracle (GPU)."""
import numpy as np
import pytest

from inner_cases import random_inputs
from oracle import lq_assemble as orc


def test_oracle_hand_case():
    """nx=2 nu=1 nc=2 (one equality row, one inactive negative-orthant row), N=1: every entry
    checked against numbers worked out by hand from solver-proxddp.hxx:25-69, 734-805."""
    inp = dict(Jx=np.array([[[1., 2.], [3., 4.]]]), Ju=np.array([[[5.], [6.]]]), slack=np.array([[.5, -.5]]),
               Lxx=np.array([[[2., 1.], [1., 3.]]]), Lxu=np.array([[[1.], [0.]]]), Luu=np.array([[[4.]]]),
               Lx=np.array([[1., 1.]]), Lu=np.array([[2.]]),
               cJx=np.array([[[1., 0.], [0., 2.]]]), cJu=np.array([[[1.], [3.]]]), Lv=np.array([[2., 4.]]),
               shifted=np.array([[0.3, -1.0]]), lo=np.array([np.inf, -np.inf]), hi=np.array([np.inf, 0.0]),
               Lxx_N=np.eye(2), Lx_N=np.array([1., 2.]), G0=-np.eye(2), g0=np.array([.1, .2]),
               Hxx0=np.array([[10., 0.], [0., 10.]]), preg=0.5, mu_inv=10.0)
    p = orc.assemble_problem(inp, 1, 2, 1, 2, 0, 2)
    k = p["stages"][0]
    assert np.array_equal(k["A"], inp["Jx"][0]) and np.array_equal(k["B"], inp["Ju"][0])
    assert np.array_equal(k["f"], [.5, -.5])
    assert np.array_equal(k["Q"], [[12.5, 1.], [1., 13.5]])      # Lxx + preg I + Hxx0
    assert np.array_equal(k["R"], [[4.5]]) and np.array_equal(k["S"], [[1.], [0.]])
    # row 0 (equality) active -> kept; row 1: shifted = -1 <= 0 -> inactive -> zeroed
    assert np.array_equal(k["C"], [[1., 0.], [0., 0.]]) and np.array_equal(k["D"], [[1.], [0.]])
    assert np.array_equal(k["d"], [2., 4.])
    # corrections: (P - Ptilde)^T (Lv * mu_inv) = row 1 only: [0, 2]*40, [3]*40
    assert np.allclose(k["q"], [1. + 0., 1. + 80.]) and np.allclose(k["r"], [2. + 120.])
    assert np.array_equal(p["term"]["Q"], 1.5 * np.eye(2)) and np.array_equal(p["term"]["q"], [1., 2.])
    assert np.array_equal(p["G0"], -np.eye(2)) and np.array_equal(p["g0"], [.1, .2])


def test_oracle_pack_matches_product_layout():
    import aligator_b200.gar as gar
    from aligator_b200.lqr import LqrKnot
    rng = np.random.default_rng(0)
    N, nx, nu, nc, nct, nc0 = 3, 3, 2, 2, 1, 3
    p = orc.assemble_problem(random_inputs(rng, N, nx, nu, nc, nct, nc0), N, nx, nu, nc, nct, nc0)
    srec = gar.stage_record_doubles(nx, nu, nc)
    stage, term, G0, g0 = orc.pack(p, N, nx, nu, nc, nct, srec)
    k = LqrKnot(nx, nu, nc)
    for n in ("A", "B", "f", "Q", "S", "R", "q", "r", "C", "D", "d"):
        getattr(k, n)[...] = p["stages"][1][n]
    assert np.array_equal(gar.pack_stage_knot(k, srec), stage[1])
    assert term.size == gar.term_record_doubles(nx, nct)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(5, 12, 6, 0, 0, 12, 7, True), (6, 4, 2, 2, 3, 4, 33, True),
                                   (3, 7, 3, 5, 0, 0, 5, False), (0, 4, 2, 0, 2, 4, 3, True),
                                   (4, 57, 28, 0, 0, 57, 2, True)])
def test_cuda_assembly_matches_oracle(shape):
    """ab2_gar_assemble against the numpy restatement on identical inputs (1e-14 relative:
    copies are exact, the sums differ only in association), then the sweep on the assembled
    problem equals the sweep on the oracle-assembled, host-uploaded problem."""
    import torch
    import __graft_entry__ as g
    g.build()
    import aligator_b200.gar as gar
    N, nx, nu, nc, nct, nc0, B, exact = shape
    rng = np.random.default_rng(sum(shape[:6]))
    per = [random_inputs(rng, N, nx, nu, nc, nct, nc0, exact=exact, init_hess=(N > 0)) for _ in range(B)]
    preg, mu_inv = per[0]["preg"], per[0]["mu_inv"]
    for q in per:
        q["preg"], q["mu_inv"] = preg, mu_inv
        for n in ("lo", "hi", "loN", "hiN"):
            if n in per[0]:
                q[n] = per[0][n]
    srec = gar.stage_record_doubles(nx, nu, nc)
    packed = [orc.pack(orc.assemble_problem(q, N, nx, nu, nc, nct, nc0), N, nx, nu, nc, nct, srec) for q in per]
    want = [np.stack([p[i] for p in packed]) for i in range(4)]
    dev = {}
    shared = ("lo", "hi", "loN", "hiN")
    for n in gar._LQ_PTRS:
        if n in per[0] and per[0][n] is not None:
            a = per[0][n] if n in shared else np.stack([q[n] for q in per])
            # blocks are column-major: transpose the trailing two axes of matrices
            if a.ndim >= 2 and n not in shared and n in ("Jx", "Ju", "Lxx", "Lxu", "Luu", "Hxx", "Hxu", "Huu",
                                                         "cJx", "cJu", "Lxx_N", "cJx_N", "G0", "Hxx0"):
                a = np.swapaxes(a, -1, -2)
            dev[n] = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    s.assemble(dev, preg, mu_inv)
    s.synchronize()
    for i in range(4):
        if want[i].size == 0:
            continue
        got = s.get_problem(i).reshape(want[i].shape)
        scale = np.abs(want[i]).max() + 1e-300
        err = np.max(np.abs(got - want[i]))
        assert err <= 1e-13 * scale, (("stage", "term", "G0", "g0")[i], err, scale)
    # the assembled problem is the solver's current problem: sweep it and compare
    mueq = 1.0 / mu_inv
    s.sweep(mueq)
    xs = s.get(gar.OUT_XS)
    fb = s.get(gar.OUT_FB)
    s2 = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    s2.set_problem(*want)
    s2.sweep(mueq)
    assert np.all(s.status() == s2.status())
    ok = s2.status() == 0
    assert np.allclose(xs[ok], s2.get(gar.OUT_XS)[ok], rtol=1e-9, atol=1e-9)
    if N > 0:
        assert np.allclose(fb[ok], s2.get(gar.OUT_FB)[ok], rtol=1e-9, atol=1e-9)
    s.close()
    s2.close()
