"""The tangent (forward mode) of the LQ solve on the CPU: the oracle's solve of the tangent problem built by the numpy
restatement (lq_tangent_ref.py) against central finite differences of the dense solve, against -K^-1 (Kdot z + hdot)
of the dense KKT system, and against the adjoint through the duality <zbar, zdot> = <grad, pdot>; and the symmetric
part of an asymmetric Q / R tangent."""
import numpy as np
import pytest

import gen
import lq_adjoint_ref as aref
import lq_tangent_ref as ref
from oracle import gar_oracle as orc

MU = 1e-2
STAGE_BLOCKS = ("A", "B", "f", "Q", "S", "R", "q", "r", "C", "D", "d")
TERM_BLOCKS = ("Q", "q", "C", "d")

# (nx, nu, nc, nct, nc0, N)
CASES = [(3, 2, 1, 1, 3, 4), (3, 2, 0, 0, 1, 1), (4, 2, 1, 0, 0, 4), (4, 3, 0, 1, 4, 0), (5, 2, 1, 1, 1, 4),
         (5, 2, 0, 0, 5, 1), (4, 2, 1, 1, 0, 1), (3, 1, 1, 1, 1, 0), (5, 3, 1, 0, 0, 0), (4, 2, 0, 1, 1, 4)]
IDS = ["nx%d_nu%d_nc%d_nct%d_nc0%d_N%d" % c for c in CASES]


def _problem(case, seed):
    nx, nu, nc, nct, nc0, N = case
    p = gen.generate_batch(seed, 1, N, nx, nu, nc, nct)
    return gen.general_initial_condition(p, nc0, seed)[0]


def _records(p, case):
    """Packed (padded) single-instance records of problem p."""
    nx, nu, nc, nct, nc0, N = case
    _, srec = aref.stage_offsets(nx, nu, nc)
    stage = np.zeros((1, N, srec))
    for t in range(N):
        r = gen.stage_record(p.stages[t])
        stage[0, t, :r.size] = r
    return (stage, gen.term_record(p.stages[N])[None], np.asarray(p.G0).ravel(order="F")[None],
            np.asarray(p.g0)[None])


def _symmetrize(rec, off, n):
    a, b = off
    M = rec[..., a:b].reshape(*rec.shape[:-1], n, n)
    rec[..., a:b] = (0.5 * (M + np.swapaxes(M, -1, -2))).reshape(*rec.shape[:-1], n * n)


def _tangent(case, seed, symmetric, pad=0.0):
    """A random data tangent; `symmetric`: Qdot, Rdot and Qdot_N symmetric.  `pad`: the value of the pad double."""
    nx, nu, nc, nct, nc0, N = case
    rng = np.random.default_rng(seed + 2000)
    so, srec = aref.stage_offsets(nx, nu, nc)
    to, trec = aref.term_offsets(nx, nct)
    st = rng.standard_normal((1, N, srec))
    st[..., so["d"][1]:] = pad
    tt = rng.standard_normal((1, trec))
    if symmetric:
        _symmetrize(st, so["Q"], nx)
        _symmetrize(st, so["R"], nu)
        _symmetrize(tt, to["Q"], nx)
    return dict(stage=st, term=tt, G0=rng.standard_normal((1, nc0 * nx)), g0=rng.standard_normal((1, nc0)))


def _dense(p):
    k0, kN = p.stages[0], p.stages[-1]
    N = p.horizon
    dims = (kN.nx, k0.nu if N else 0, k0.nc if N else 0, kN.nc, p.nc0, N)
    return aref.solution_dict([gen.lqr_dense_solve(p, MU)], dims)


def _oracle_solve(recs, case):
    nx, nu, nc, nct, nc0, N = case
    bo = orc.BatchedOracle(nx, nu, nc, nct, nc0, N, 1, *[np.ascontiguousarray(a) for a in recs])
    bo.sweep(MU, nthreads=1)
    assert np.all(bo.status == 1)  # the oracle reports 1 = ok
    return aref.oracle_dict(bo.get())


def _oracle_tangent(p, case, dot):
    recs = _records(p, case)
    z = _oracle_solve(recs, case)
    return _oracle_solve(ref.tangent_records(*recs, dot, z, case), case)


def _with_blocks(p, case, dot, h):
    """A copy of problem p with every block moved by h times the tangent's block."""
    nx, nu, nc, nct, nc0, N = case
    so, _ = aref.stage_offsets(nx, nu, nc)
    to, _ = aref.term_offsets(nx, nct)
    q = p.copy()
    put = lambda k, n, rec, off: setattr(k, n, np.asarray(getattr(k, n), dtype=np.float64)
                                         + h * rec[off[0]:off[1]].reshape(np.shape(getattr(k, n)), order="F"))
    for t in range(N):
        for n in STAGE_BLOCKS:
            put(q.stages[t], n, dot["stage"][0, t], so[n])
    for n in TERM_BLOCKS:
        put(q.stages[N], n, dot["term"][0], to[n])
    q.G0 = np.asarray(p.G0, dtype=np.float64) + h * dot["G0"][0].reshape(nc0, nx, order="F")
    q.g0 = np.asarray(p.g0, dtype=np.float64) + h * dot["g0"][0]
    return q


def _zero_blocks(p):
    """A copy of problem p with every block zero."""
    q = p.copy()
    for k in q.stages:
        for n in STAGE_BLOCKS:
            if hasattr(k, n):
                setattr(k, n, np.zeros(np.shape(getattr(k, n))))
    q.G0, q.g0 = np.zeros(np.shape(p.G0)), np.zeros(np.shape(p.g0))
    return q


def _split(p, vec):
    """A vector in the dense KKT system's unknown order -> solution dict."""
    nx, N, nc0 = p.stages[-1].nx, p.horizon, p.nc0
    _, _, offs = gen.lqr_dense_kkt(p, MU)
    st = p.stages
    xs = [vec[o:o + m.nx] for o, m in zip(offs, st)]
    us = [vec[o + m.nx:o + m.nx + m.nu] for o, m in zip(offs[:N], st[:N])]
    vs = [vec[o + m.nx + m.nu:o + m.nx + m.nu + m.nc] for o, m in zip(offs, st)]
    lb = [vec[:nc0]] + [vec[o + m.nx + m.nu + m.nc:o + 2 * m.nx + m.nu + m.nc] for o, m in zip(offs[:N], st[:N])]
    dims = (nx, st[0].nu if N else 0, st[0].nc if N else 0, st[N].nc, nc0, N)
    return aref.solution_dict([(xs, us + [np.zeros(0)], vs, lb)], dims)


def _check(got, want, tol, tag):
    for k in aref.KEYS:
        if np.asarray(want[k]).size:
            e = gen.rel_fro(got[k], want[k])
            assert e <= tol, (tag, k, e)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_tangent_matches_finite_differences(case):
    seed = sum(c * 7 ** i for i, c in enumerate(case))
    p = _problem(case, seed)
    dot = _tangent(case, seed, symmetric=True)
    h = 1e-6
    zp, zm = _dense(_with_blocks(p, case, dot, h)), _dense(_with_blocks(p, case, dot, -h))
    fd = {k: (zp[k] - zm[k]) / (2 * h) for k in aref.KEYS}
    _check(_oracle_tangent(p, case, dot), fd, 1e-6, "fd")


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_tangent_matches_dense_kkt(case):
    """zdot = -K^-1 (Kdot z + hdot), with Kdot and hdot the dense system of the tangent's blocks (K is affine)."""
    seed = sum(c * 5 ** i for i, c in enumerate(case))
    p = _problem(case, seed)
    dot = _tangent(case, seed, symmetric=True)
    K, rhs, _ = gen.lqr_dense_kkt(p, MU)
    z = np.linalg.solve(K, -rhs)
    zero = _zero_blocks(p)
    Kd, hd, _ = gen.lqr_dense_kkt(_with_blocks(zero, case, dot, 1.0), 0.0)
    K0, _, _ = gen.lqr_dense_kkt(zero, 0.0)  # the constant -I couplings of the dynamics
    zdot = -np.linalg.solve(K, (Kd - K0) @ z + hd)
    # the tangent problem is built at the same z: the primal's own error (up to 1e-13 here) would otherwise enter rho
    recs = _records(p, case)
    got = _oracle_solve(ref.tangent_records(*recs, dot, _split(p, z), case), case)
    _check(got, _split(p, zdot), 1e-12, "dense")


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_duality_with_the_adjoint(case):
    """<zbar, zdot> = <grad(zbar), pdot> for an asymmetric Qdot, Rdot, Qdot_N and a nonzero pad double."""
    seed = sum(c * 3 ** i for i, c in enumerate(case))
    p = _problem(case, seed)
    dot = _tangent(case, seed, symmetric=False, pad=3.0)
    rng = np.random.default_rng(seed + 3000)
    zbar = {k: rng.standard_normal(s) for k, s in aref._shapes(case, 1).items()}
    recs = _records(p, case)
    z = _oracle_solve(recs, case)
    zdot = _oracle_solve(ref.tangent_records(*recs, dot, z, case), case)
    w = _oracle_solve(aref.adjoint_records(*recs, zbar, case), case)
    grad = aref.grad_records(z, w, case)
    lhs = sum(float(np.sum(zbar[k] * zdot[k])) for k in aref.KEYS)
    rhs = sum(float(np.sum(grad[k] * dot[k])) for k in ("stage", "term", "G0", "g0"))
    assert abs(lhs - rhs) <= 1e-12 * max(abs(lhs), abs(rhs)), (lhs, rhs)


@pytest.mark.parametrize("case", [CASES[0], CASES[4], CASES[9]], ids=[IDS[0], IDS[4], IDS[9]])
def test_asymmetric_q_and_r_act_as_their_symmetric_part(case):
    nx, nu, nc, nct, nc0, N = case
    p = _problem(case, 11)
    dot = _tangent(case, 11, symmetric=False)
    sym = {k: v.copy() for k, v in dot.items()}
    so, _ = aref.stage_offsets(nx, nu, nc)
    to, _ = aref.term_offsets(nx, nct)
    _symmetrize(sym["stage"], so["Q"], nx)
    _symmetrize(sym["stage"], so["R"], nu)
    _symmetrize(sym["term"], to["Q"], nx)
    assert not np.array_equal(sym["stage"], dot["stage"])
    a, b = _oracle_tangent(p, case, dot), _oracle_tangent(p, case, sym)
    for k in aref.KEYS:
        assert np.array_equal(a[k], b[k]), k


def test_null_tangent_fields_are_zero():
    case = (4, 2, 1, 1, 4, 2)
    p = _problem(case, 3)
    recs = _records(p, case)
    z = _oracle_solve(recs, case)
    dot = _tangent(case, 3, symmetric=False)
    for drop in (("stage",), ("term", "g0"), ("G0",), ("stage", "term", "G0", "g0")):
        part = {k: (None if k in drop else v) for k, v in dot.items()}
        expl = {k: (np.zeros_like(v) if k in drop else v) for k, v in dot.items()}
        a, b = ref.rho(part, z, case), ref.rho(expl, z, case)
        for k in aref.KEYS:
            assert np.array_equal(a[k], b[k]), (drop, k)
    st, tt, G0, g0 = ref.tangent_records(*recs, {}, z, case)
    so, _ = aref.stage_offsets(4, 2, 1)
    for n in ("f", "q", "r", "d"):
        assert not np.any(st[..., so[n][0]:so[n][1]])
    assert np.array_equal(G0, recs[2]) and not np.any(g0)
