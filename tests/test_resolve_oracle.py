"""ab2_gar_resolve on the CPU: the numpy restatement of the kernel's algebra (lq_resolve_ref.py), fed with the
oracle's factorisation, against the oracle's full solve of the problem with its vectors replaced, against the dense
KKT solve, and through the identities resolve(own vectors) = primal, resolve(-zbar) = adjoint, resolve(rho) = tangent;
and the device program itself, compiled for the host and run on emulated lanes (tests/emu/resolve_emu.cpp), against
the restatement."""
import ctypes as C
import os

import numpy as np
import pytest

import emu_harness
import gen
import lq_adjoint_ref as aref
import lq_resolve_ref as ref
import lq_tangent_ref as tref
from emu_harness import run_resolve
from lq_cases import BAR_CASES, bar_case, bar_violations, batch_records
from oracle import gar_oracle as orc

MU = 1e-2
HERE = os.path.dirname(os.path.abspath(__file__))

# (nx, nu, nc, nct, nc0, N): C1, C2 and C3 dims, nct > 0, nc0 in {0, 1, nx/2, nx}, N in {0, 1, 100}
CASES = [(6, 3, 0, 0, 6, 4), (6, 3, 0, 2, 3, 1), (12, 6, 0, 0, 12, 3), (12, 6, 0, 3, 1, 0), (4, 2, 2, 2, 4, 5),
         (4, 2, 2, 0, 0, 1), (4, 2, 2, 2, 2, 100), (5, 2, 1, 1, 0, 0), (6, 3, 0, 0, 6, 100), (12, 6, 0, 0, 6, 1)]
IDS = ["nx%d_nu%d_nc%d_nct%d_nc0%d_N%d" % c for c in CASES]


def _batch(case, seed, B=2, mutate=None):
    nx, nu, nc, nct, nc0, N = case
    probs = gen.general_initial_condition(gen.generate_batch(seed, B, N, nx, nu, nc, nct), nc0, seed)
    if mutate:
        probs = mutate(probs)
    return probs


def _oracle(recs, case, mu=MU):
    nx, nu, nc, nct, nc0, N = case
    B = recs[1].shape[0]
    bo = orc.BatchedOracle(nx, nu, nc, nct, nc0, N, B, *[np.ascontiguousarray(a) for a in recs])
    bo.sweep(mu, nthreads=1)
    assert np.all(bo.status == 1)
    return bo.get()


def _resolve_ref(recs, o, h, case, nrhs, mu=MU):
    stage, term, G0, _ = recs
    return ref.resolve(stage, term, G0, o["fb"], o["fbT"], o["Vxx"], h, case, mu, nrhs)


def _pick(z, j):
    return {k: v[j] for k, v in z.items()}


def _assert_close(z, want, tol, what=""):
    for k in ref.SOL:
        assert gen.rel_fro(z[k], want[k]) <= tol, (what, k, gen.rel_fro(z[k], want[k]))


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_matches_oracle_and_dense_solve_of_replaced_problem(case):
    recs = batch_records(_batch(case, 11), case)
    o = _oracle(recs, case)
    B, nrhs = 2, 3
    h = ref.random_rhs(np.random.default_rng(5), case, B, nrhs)
    z = _resolve_ref(recs, o, h, case, nrhs)
    for j in range(nrhs):
        hj = {k: v[j] for k, v in h.items()}
        want = aref.oracle_dict(_oracle(ref.replaced_records(*recs, hj, case), case))
        _assert_close(_pick(z, j), want, 1e-12, "oracle rhs %d" % j)
    # dense KKT solve of the replaced problems (rhs 0)
    stage, term, G0, g0 = ref.replaced_records(*recs, {k: v[0] for k, v in h.items()}, case)
    nx, nu, nc, nct, nc0, N = case
    probs = _batch(case, 11)
    so, _ = aref.stage_offsets(nx, nu, nc)
    to, _ = aref.term_offsets(nx, nct)
    sols = []
    for b, p in enumerate(probs):
        for t in range(N):
            k = p.stages[t]
            for name in ("q", "r", "f", "d"):
                getattr(k, name)[:] = stage[b, t, so[name][0]:so[name][1]]
        p.stages[N].q[:] = term[b, to["q"][0]:to["q"][1]]
        p.stages[N].d[:] = term[b, to["d"][0]:to["d"][1]]
        p.g0[:] = g0[b]
        sols.append(gen.lqr_dense_solve(p, MU))
    _assert_close(_pick(z, 0), aref.solution_dict(sols, case), 1e-12, "dense")


@pytest.mark.parametrize("case", CASES[:6], ids=IDS[:6])
def test_identities(case):
    nx, nu, nc, nct, nc0, N = case
    recs = batch_records(_batch(case, 12), case)
    stage, term, G0, g0 = recs
    o = _oracle(recs, case)
    primal = aref.oracle_dict(o)
    B = 2
    rng = np.random.default_rng(6)
    # linearity
    h1, h2 = ref.random_rhs(rng, case, B, 1), ref.random_rhs(rng, case, B, 1)
    z1, z2 = _resolve_ref(recs, o, h1, case, 1), _resolve_ref(recs, o, h2, case, 1)
    z12 = _resolve_ref(recs, o, {k: 2.0 * h1[k] - 0.5 * h2[k] for k in h1}, case, 1)
    _assert_close(z12, {k: 2.0 * z1[k] - 0.5 * z2[k] for k in z1}, 1e-12, "linearity")
    # the problem's own vectors give the primal
    so, _ = aref.stage_offsets(nx, nu, nc)
    to, _ = aref.term_offsets(nx, nct)
    vec = lambda name: stage[..., so[name][0]:so[name][1]]
    q = np.concatenate([vec("q"), term[:, None, to["q"][0]:to["q"][1]]], axis=1)
    own = dict(q=q, r=vec("r"), d=vec("d"), dN=term[:, to["d"][0]:to["d"][1]], g0=g0, f=vec("f"))
    _assert_close(_pick(_resolve_ref(recs, o, {k: v[None] for k, v in own.items()}, case, 1), 0), primal, 1e-12,
                  "primal")
    # h = -zbar gives the adjoint's w
    zbar = {k: rng.standard_normal(v.shape) for k, v in primal.items()}
    w = aref.oracle_dict(_oracle(aref.adjoint_records(*recs, zbar, case), case))
    hb = dict(q=-zbar["xs"], r=-zbar["us"], d=-zbar["vs"], dN=-zbar["vsT"], g0=-zbar["lam0"], f=-zbar["lams"])
    _assert_close(_pick(_resolve_ref(recs, o, {k: v[None] for k, v in hb.items()}, case, 1), 0), w, 1e-12, "adjoint")
    # h = rho gives the tangent
    _, srec = aref.stage_offsets(nx, nu, nc)
    _, trec = aref.term_offsets(nx, nct)
    dot = dict(stage=rng.standard_normal((B, N, srec)), term=rng.standard_normal((B, trec)),
               G0=rng.standard_normal((B, nc0 * nx)), g0=rng.standard_normal((B, nc0)))
    zdot = aref.oracle_dict(_oracle(tref.tangent_records(*recs, dot, primal, case), case))
    rho = tref.rho(dot, primal, case)
    hr = dict(q=rho["xs"], r=rho["us"], d=rho["vs"], dN=rho["vsT"], g0=rho["lam0"], f=rho["lams"])
    _assert_close(_pick(_resolve_ref(recs, o, {k: v[None] for k, v in hr.items()}, case, 1), 0), zdot, 1e-11,
                  "tangent")


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_emulation_matches_restatement(case):
    recs = batch_records(_batch(case, 13), case)
    o = _oracle(recs, case)
    B, nrhs = 2, 3
    h = ref.random_rhs(np.random.default_rng(7), case, B, nrhs)
    want = _resolve_ref(recs, o, h, case, nrhs)
    runs = [(32, 3, False, 0), (5, 2, True, 1)] if case[5] < 100 else [(32, 2, True, 0)]
    for lanes, chunk, packed, head in runs:
        z = run_resolve(recs, o, h, case, nrhs, MU, lanes, chunk, packed, head)
        _assert_close(z, want, 1e-12, (lanes, chunk, packed, head))


def test_emulation_bit_equal_across_chunks_and_lanes():
    case = (4, 2, 2, 2, 2, 5)
    recs = batch_records(_batch(case, 14), case)
    o = _oracle(recs, case)
    nrhs = 5
    h = ref.random_rhs(np.random.default_rng(8), case, 2, nrhs)
    base = run_resolve(recs, o, h, case, nrhs, MU, 32, nrhs, True, 0)
    for lanes, chunk in ((32, 1), (7, 2), (3, 4)):
        z = run_resolve(recs, o, h, case, nrhs, MU, lanes, chunk, True, 0)
        for k in ref.SOL:
            assert np.array_equal(z[k], base[k]), (lanes, chunk, k)
    # one right-hand side alone equals its place among five
    one = run_resolve(recs, o, {k: v[3:4] for k, v in h.items()}, case, 1, MU, 32, 1, True, 0)
    for k in ref.SOL:
        assert np.array_equal(one[k][0], base[k][3]), k


@pytest.mark.parametrize("mutate,case", [(gen.make_2x2_pivots, (4, 2, 2, 2, 4, 6)),
                                         (gen.make_pivoting, (6, 3, 0, 0, 6, 6))], ids=["2x2", "interchange"])
def test_emulation_forced_pivots(mutate, case):
    recs = batch_records(_batch(case, 15, mutate=mutate), case)
    # the 2x2 case's KKT condition number grows like 1/mu: two correct fp64 solvers differ by about cond * u
    for mu, tol in ((1e-3, 1e-11), (1e-8, 1e-6)):
        o = _oracle(recs, case, mu)
        h = ref.random_rhs(np.random.default_rng(9), case, 2, 2)
        z = run_resolve(recs, o, h, case, 2, mu, 32, 2, True, 0)
        _assert_close(z, _resolve_ref(recs, o, h, case, 2, mu), tol, mu)
        for j in range(2):
            oracle = aref.oracle_dict(_oracle(ref.replaced_records(*recs, {k: v[j] for k, v in h.items()}, case),
                                              case, mu))
            _assert_close(_pick(z, j), oracle, tol, ("oracle", mu, j))


def test_every_served_shape_fits_shared_memory():
    """Every shape a plain serial handle accepts (ab2_gar_supported, compile-time or CTA-per-instance kernel) runs one
    right-hand side per warp within 227 KB of shared memory."""
    from aligator_b200 import gar
    fn = C.CFUNCTYPE(C.c_int, C.c_int, C.c_int, C.c_int, C.c_int)(("ab2_gar_supported", gar.lib()))
    bad = (C.c_int * 6)()
    largest, accepted = C.c_long(), C.c_long()
    e = emu_harness.lib()
    over = e.emu_item_size_scan(e.emu_resolve_item_bytes, 0, C.cast(fn, C.c_void_p), 130, bad, C.byref(largest),
                                C.byref(accepted))
    assert over == 0, (over, list(bad))
    assert 0 < largest.value <= 227 * 1024


@pytest.mark.parametrize("name", list(BAR_CASES))
def test_emulation_meets_the_conditioning_bar(name):
    probs, recs, case, mu, h = bar_case(name)
    z = run_resolve(recs, _oracle(recs, case, mu), h, case, 2, mu, 32, 2, True, 0)
    for j in range(2):
        bad, tab = bar_violations(probs, recs, case, mu, {k: v[j] for k, v in h.items()}, _pick(z, j))
        assert not bad, "%s rhs %d\n%s" % (name, j, tab)
