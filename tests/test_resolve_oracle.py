"""ab2_gar_resolve on the CPU: the numpy restatement of the kernel's algebra (lq_resolve_ref.py), fed with the
oracle's factorisation, against the oracle's full solve of the problem with its vectors replaced, against the dense
KKT solve, and through the identities resolve(own vectors) = primal, resolve(-zbar) = adjoint, resolve(rho) = tangent;
and the device program itself, compiled for the host and run on emulated lanes (tests/emu/resolve_emu.cpp), against
the restatement."""
import ctypes as C
import functools
import os

import numpy as np
import pytest

import emu_harness
import gen
import lq_adjoint_ref as aref
import lq_resolve_ref as ref
import lq_tangent_ref as tref
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


def _records(probs, case):
    nx, nu, nc, nct, nc0, N = case
    _, srec = aref.stage_offsets(nx, nu, nc)
    B = len(probs)
    stage = np.zeros((B, N, srec))
    for b, p in enumerate(probs):
        for t in range(N):
            r = gen.stage_record(p.stages[t])
            stage[b, t, :r.size] = r
    term = np.stack([gen.term_record(p.stages[N]) for p in probs])
    G0 = np.stack([np.asarray(p.G0).ravel(order="F") for p in probs]).reshape(B, nc0 * nx)
    g0 = np.stack([np.asarray(p.g0) for p in probs]).reshape(B, nc0)
    return stage, term, G0, g0


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
    recs = _records(_batch(case, 11), case)
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
    recs = _records(_batch(case, 12), case)
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


# ---- host emulation of the device program ----
@functools.lru_cache(maxsize=None)
def _emu():
    h = emu_harness.lib()
    h.emu_resolve.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
    return h


def _pack_vxx(Vxx):
    """[B][N+1][nx][nx] (row index first) -> the packed layout of vxx_layout.h: packed lower triangles, and the full
    column-major slot-0 blocks."""
    B, K, nx, _ = Vxx.shape
    P = (nx * (nx + 1) // 2 + 1) & ~1
    pk = np.zeros((B, K, P))
    for j in range(nx):
        c0 = j * nx - j * (j - 1) // 2
        pk[:, :, c0:c0 + nx - j] = Vxx[:, :, j:, j]
    return pk, np.ascontiguousarray(np.swapaxes(Vxx[:, 0], -1, -2)).reshape(B, nx * nx)


def _run_emu(recs, o, h, case, nrhs, mu, lanes, chunk, packed, head):
    nx, nu, nc, nct, nc0, N = case
    stage, term, G0, _ = recs
    B = term.shape[0]
    if head and N:
        stage = np.roll(stage, head, axis=1)  # knot t in slot (t + head) mod N
    Vxx = np.asarray(o["Vxx"])
    if packed:
        V, V0 = _pack_vxx(Vxx)
    else:
        V, V0 = np.ascontiguousarray(np.swapaxes(Vxx, -1, -2)), None
    keep = [np.ascontiguousarray(a, dtype=np.float64) for a in (stage, term, G0, o["fb"], o["fbT"], V)]
    keep.append(None if V0 is None else np.ascontiguousarray(V0))
    hf = ref.full_rhs(h, case, B, nrhs)
    keep += [np.ascontiguousarray(hf[k]) for k in ref.RHS]
    out = {k: np.full((nrhs,) + s, np.nan) for k, s in zip(ref.SOL, ref.rhs_shapes(case, B).values())}
    ptr = lambda a: None if a is None or a.size == 0 else a.ctypes.data
    ins = (C.c_void_p * 13)(*[ptr(a) for a in keep])
    outs = (C.c_void_p * 6)(*[ptr(out[k]) for k in ref.SOL])
    _, srec = aref.stage_offsets(nx, nu, nc)
    dims = np.array([B, N, nx, nu, nc, nct, nc0, srec, term.shape[1], head if N else 0, nrhs, chunk, lanes],
                    dtype=np.int32)
    mub = None if np.ndim(mu) == 0 else np.ascontiguousarray(mu, dtype=np.float64)
    _emu().emu_resolve(dims.ctypes.data, float(mu) if mub is None else 0.0, ptr(mub), ins, outs)
    return out


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_emulation_matches_restatement(case):
    recs = _records(_batch(case, 13), case)
    o = _oracle(recs, case)
    B, nrhs = 2, 3
    h = ref.random_rhs(np.random.default_rng(7), case, B, nrhs)
    want = _resolve_ref(recs, o, h, case, nrhs)
    runs = [(32, 3, False, 0), (5, 2, True, 1)] if case[5] < 100 else [(32, 2, True, 0)]
    for lanes, chunk, packed, head in runs:
        z = _run_emu(recs, o, h, case, nrhs, MU, lanes, chunk, packed, head)
        _assert_close(z, want, 1e-12, (lanes, chunk, packed, head))


def test_emulation_bit_equal_across_chunks_and_lanes():
    case = (4, 2, 2, 2, 2, 5)
    recs = _records(_batch(case, 14), case)
    o = _oracle(recs, case)
    nrhs = 5
    h = ref.random_rhs(np.random.default_rng(8), case, 2, nrhs)
    base = _run_emu(recs, o, h, case, nrhs, MU, 32, nrhs, True, 0)
    for lanes, chunk in ((32, 1), (7, 2), (3, 4)):
        z = _run_emu(recs, o, h, case, nrhs, MU, lanes, chunk, True, 0)
        for k in ref.SOL:
            assert np.array_equal(z[k], base[k]), (lanes, chunk, k)
    # one right-hand side alone equals its place among five
    one = _run_emu(recs, o, {k: v[3:4] for k, v in h.items()}, case, 1, MU, 32, 1, True, 0)
    for k in ref.SOL:
        assert np.array_equal(one[k][0], base[k][3]), k


@pytest.mark.parametrize("mutate,case", [(gen.make_2x2_pivots, (4, 2, 2, 2, 4, 6)),
                                         (gen.make_pivoting, (6, 3, 0, 0, 6, 6))], ids=["2x2", "interchange"])
def test_emulation_forced_pivots(mutate, case):
    recs = _records(_batch(case, 15, mutate=mutate), case)
    # the 2x2 case's KKT condition number grows like 1/mu: two correct fp64 solvers differ by about cond * u
    for mu, tol in ((1e-3, 1e-11), (1e-8, 1e-6)):
        o = _oracle(recs, case, mu)
        h = ref.random_rhs(np.random.default_rng(9), case, 2, 2)
        z = _run_emu(recs, o, h, case, 2, mu, 32, 2, True, 0)
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
    bad = (C.c_int * 4)()
    largest = C.c_long()
    e = _emu()
    e.emu_resolve_size_scan.restype = C.c_long
    e.emu_resolve_size_scan.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    over = e.emu_resolve_size_scan(C.cast(fn, C.c_void_p), 130, bad, C.byref(largest))
    assert over == 0, (over, list(bad))
    assert 0 < largest.value <= 227 * 1024


# ---- the conditioning bar of DESIGN §5: against the extended-precision solve of each replaced problem ----
TRAJ = ("xs", "us", "vs", "lbd")
# name: ((nx, nu, nc, nct, N), B, mu, transform)
BAR_CASES = {
    "c3_mu1e-3": ((4, 2, 2, 0, 20), 3, 1e-3, None),
    "c3_mu1e-8": ((4, 2, 2, 0, 30), 3, 1e-8, None),
    "c3_mu1e-11": ((4, 2, 2, 0, 30), 3, 1e-11, None),
    "c3_nct_mu1e-8": ((4, 2, 2, 2, 10), 2, 1e-8, None),
    "pivots_2x2_mu1e-3": ((4, 2, 2, 0, 10), 2, 1e-3, gen.make_2x2_pivots),
    "pivots_2x2_mu1e-8": ((4, 2, 2, 0, 10), 2, 1e-8, gen.make_2x2_pivots),
    "interchanges": ((12, 6, 0, 0, 8), 2, 1e-8, gen.make_pivoting),
}


def bar_case(name):
    """(problems, packed records, dims, mu, right-hand sides [2][B][...])."""
    (nx, nu, nc, nct, N), B, mu, transform = BAR_CASES[name]
    probs = gen.generate_batch(3000 + sum(map(ord, name)), B, N, nx, nu, nc, nct)
    if transform is not None:
        transform(probs)
    case = (nx, nu, nc, nct, nx, N)
    return probs, _records(probs, case), case, mu, ref.random_rhs(np.random.default_rng(len(name)), case, B, 2)


def bar_violations(probs, recs, case, mu, hj, got):
    """Families of the trajectory where `got` (one right-hand side's solution dict) is further from the extended-precision
    solve of the replaced problem than max(16 e_oracle, 64 u) allows."""
    import hp_reference as hp
    nx, nu, nc, nct, nc0, N = case
    want, _ = hp.solve(ref.replaced_problems(probs, hj), mu)
    e_oracle = hp.error_families(_oracle(ref.replaced_records(*recs, hj, case), case, mu), want, nu, nc, N, TRAJ)
    z = dict(got, lbd0=got["lam0"], lbdas=got["lams"])
    e_kernel = hp.error_families(z, want, nu, nc, N, TRAJ)
    return hp.violations(e_kernel, e_oracle), hp.table("", e_oracle, e_kernel)


@pytest.mark.parametrize("name", list(BAR_CASES))
def test_emulation_meets_the_conditioning_bar(name):
    probs, recs, case, mu, h = bar_case(name)
    z = _run_emu(recs, _oracle(recs, case, mu), h, case, 2, mu, 32, 2, True, 0)
    for j in range(2):
        bad, tab = bar_violations(probs, recs, case, mu, {k: v[j] for k, v in h.items()}, _pick(z, j))
        assert not bad, "%s rhs %d\n%s" % (name, j, tab)
