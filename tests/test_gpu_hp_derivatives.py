"""The derivative calls on the GPU against the extended-precision references of tests/hp_reference.py, at the bar of
DESIGN §5: e_kernel <= max(16 e_ref, 64 u) family by family, each family's error the worst per-(instance, knot)
relative error, e_ref the error of the fp64 restatement fed with the oracle's factorisation and solution
(tests/test_hp_derivatives.py).  For the dense handle e_ref is the larger of the serial oracle's and that of the
oracle's dense solver.  Calls: adjoint and tangent (and their per-instance-mu twins), adjoint_many and tangent_many,
factor_adjoint and factor_tangent; on the sweep variants, the CTA-per-instance kernels and the dense handle, and at
full-size batch counts on instances sampled across the launch."""
import functools

import numpy as np
import pytest

import gen
import hp_reference as hp
import lq_adjoint_ref as aref
import lq_factor_adjoint_ref as fadj
import lq_gpu
from aligator_b200.lqr import LqrKnot, LqrProblem
from lq_cases import Case, check_bar, run_solver, symmetric_dot

pytestmark = pytest.mark.gpu

DEFAULT, CTA, DENSE = {}, dict(variant=9), dict(dense=True)
WARP = [dict(variant=v) for v in (0, 1, 2, 3, 4, 5, 6, 7, 8, 10)]


@pytest.fixture(scope="module")
def env():
    return lq_gpu.gpu_env()


def kw_id(kw):
    return "dense" if kw.get("dense") else "v%d" % kw["variant"] if "variant" in kw else "default"


# name: ((nx, nu, nc, nct, nc0, N), batch, mu, transform, handles)
SOLVE_CASES = {
    "c3_mu1e-3": ((4, 2, 2, 0, 4, 6), 3, 1e-3, None, [DEFAULT] + WARP + [CTA, DENSE]),
    "c2_mu1e-8": ((12, 6, 0, 0, 12, 6), 2, 1e-8, None, [DEFAULT] + WARP + [CTA, DENSE]),
    "c2_nct3_mu1e-8": ((12, 6, 0, 3, 12, 5), 2, 1e-8, None, [DEFAULT, CTA, DENSE]),
    "cta_7_3_2": ((7, 3, 2, 2, 7, 5), 3, 1e-2, None, [DEFAULT]),
    "c3_N100_mu1e-8": ((4, 2, 2, 0, 4, 100), 2, 1e-8, None, [DEFAULT, CTA, DENSE]),
    "c3_N100_mu1e-11": ((4, 2, 2, 0, 4, 100), 2, 1e-11, None, [DEFAULT, CTA, DENSE]),
    "pivots_2x2": ((4, 2, 2, 2, 4, 8), 3, 1e-3, gen.make_2x2_pivots, [DEFAULT, CTA]),
    "interchanges": ((12, 6, 0, 0, 12, 6), 2, 1e-8, gen.make_pivoting, [DEFAULT, dict(variant=7), CTA]),
    "N0": ((4, 2, 2, 2, 4, 0), 2, 1e-3, None, [DEFAULT]),
    "N1": ((6, 3, 0, 2, 3, 1), 2, 1e-3, None, [DEFAULT]),
}
for _d6, _B, _mu in (((4, 2, 2, 2, 0, 6), 3, 1e-3), ((12, 6, 0, 0, 0, 3), 2, 1e-8)):
    for _nc0 in sorted({0, 1, _d6[0] // 2, _d6[0]}):
        SOLVE_CASES["G0_%d_nc0_%d" % (_d6[0], _nc0)] = (_d6[:4] + (_nc0, _d6[5]), _B, _mu, None, [DEFAULT, CTA, DENSE])
SOLVE_CASES["mu_per_instance"] = ((4, 2, 2, 2, 4, 6), 4, np.array([1e-8, 1e-5, 1e-3, 1e-1]), None, [DEFAULT])

FACTOR_CASES = {
    "c3_nct2_mu1e-3": ((4, 2, 2, 2, 4, 6), 3, 1e-3, None),
    "c3_nct2_mu1e-8": ((4, 2, 2, 2, 4, 6), 3, 1e-8, None),
    "c2_mu1e-8": ((12, 6, 0, 3, 12, 5), 2, 1e-8, None),
    "c1": ((6, 3, 0, 2, 3, 5), 3, 1e-3, None),
    "N0": ((4, 2, 2, 2, 4, 0), 2, 1e-3, None),
    "N1": ((6, 3, 0, 2, 3, 1), 2, 1e-3, None),
    "pivots_2x2": ((4, 2, 2, 2, 4, 6), 3, 1e-3, gen.make_2x2_pivots),
    "mu_per_instance": ((4, 2, 2, 2, 4, 6), 4, np.array([1e-8, 1e-5, 1e-3, 1e-1]), None),
    "c3_N100_mu1e-8": ((4, 2, 2, 2, 4, 100), 2, 1e-8, None),
}


def make_problems(d6, B, transform, seed):
    nx, nu, nc, nct, nc0, N = d6
    probs = gen.generate_batch(seed, B, N, nx, nu, nc, nct)
    gen.general_initial_condition(probs, nc0, seed)
    if transform is not None:
        transform(probs)
    return probs


def with_handle_dims(c, d6):
    """The handle's dimensions (at horizon 0 the problem has no stage knot to tell nu and nc)."""
    c.hdims = d6
    return c


@functools.lru_cache(maxsize=None)
def solve_case(name):
    d6, B, mu, transform, _ = SOLVE_CASES[name]
    return with_handle_dims(Case(make_problems(d6, B, transform, 5000 + sum(map(ord, name))), mu), d6)


@functools.lru_cache(maxsize=None)
def factor_case(name):
    d6, B, mu, transform = FACTOR_CASES[name]
    return with_handle_dims(Case(make_problems(d6, B, transform, 6000 + sum(map(ord, name))), mu), d6)


def _dense_solution(probs, d6, mu):
    nx, nu, nc, nct, nc0, N = d6
    return hp.solution_of(run_solver(probs, (nx, nu, nc, nct, N), mu, "dense"))


@functools.lru_cache(maxsize=None)
def dense_e_refs(name):
    """adjoint / tangent e_ref of the dense handle: the larger of the serial oracle's and that of the oracle's dense
    solver (its own factorisation and solution, its solves of the adjoint and tangent problems)."""
    import lq_resolve_ref as rref
    import lq_tangent_ref as tref
    c = solve_case(name)
    e = c.e_refs()
    z = _dense_solution(c.probs, c.d6, c.mu)
    neg = lambda d: dict(q=-d["xs"], r=-d["us"], d=-d["vs"], dN=-d["vsT"], g0=-d["lam0"], f=-d["lams"])
    w = _dense_solution(rref.replaced_problems(c.probs, neg(c.cot)), c.d6, c.mu)
    rho = tref.rho(c.dot, z, c.d6)
    zd = _dense_solution(rref.replaced_problems(c.probs, {k: -v for k, v in neg(rho).items()}), c.d6, c.mu)
    own = dict(adjoint=c.e_adjoint(aref.grad_records(z, w, c.d6)), tangent=c.e_tangent(zd))
    return {k: {f: max(v, e[k][f]) for f, v in own[k].items()} for k in own}


def _dev(torch, a):
    return torch.tensor(np.ascontiguousarray(a, dtype=np.float64), device="cuda")


def _devs(torch, d):
    """Device tensors of a cotangent or tangent dict; fields of zero size (the stage fields at horizon 0) as None."""
    return {k: _dev(torch, v) if np.size(v) else None for k, v in d.items()}


def _mu_arg(torch, mu):
    return mu if np.ndim(mu) == 0 else _dev(torch, mu)


def _handle(env, c, kw):
    gar, _, torch = env
    s = gar.CudaRiccatiBatch(*c.hdims, len(c.probs), **kw)
    s.set_problem(*[np.ascontiguousarray(a) for a in c.recs])
    s.sweep(_mu_arg(torch, c.mu))
    assert np.all(s.status() == 0)
    return s


def run_adjoint_tangent(env, c, kw):
    """(gradient records of adjoint, zdot of tangent) of one handle on the case's cotangent and tangent."""
    _, _, torch = env
    s = _handle(env, c, kw)
    primal = {k: v.clone() for k, v in lq_gpu.primal(env, s).items()}
    g = lq_gpu.grad_bufs(env, s)
    s.adjoint(primal, _devs(torch, c.cot), g, _mu_arg(torch, c.mu))
    s.synchronize()
    g = lq_gpu.to_np(g)
    s.tangent(primal, _devs(torch, c.dot), _mu_arg(torch, c.mu))
    s.synchronize()
    zd = lq_gpu.to_np(lq_gpu.primal(env, s))
    s.close()
    return g, zd


SOLVE_ITEMS = [(n, kw) for n in SOLVE_CASES for kw in SOLVE_CASES[n][4]]


@pytest.mark.parametrize("name,kw", SOLVE_ITEMS, ids=["%s-%s" % (n, kw_id(kw)) for n, kw in SOLVE_ITEMS])
def test_adjoint_and_tangent_meet_the_bar(env, name, kw):
    c = solve_case(name)
    e_ref = dense_e_refs(name) if kw.get("dense") else c.e_refs()
    g, zd = run_adjoint_tangent(env, c, kw)
    nx, nu, nc = c.d6[:3]
    assert np.all(g["stage"][..., aref.stage_offsets(nx, nu, nc)[0]["d"][1]:] == 0.0)  # the pad double
    e = c.e_adjoint(g)
    print("\n" + hp.table("%s %s adjoint" % (name, kw_id(kw)), e_ref["adjoint"], e))
    check_bar(e, e_ref["adjoint"], "%s %s adjoint" % (name, kw_id(kw)))
    e = c.e_tangent(zd)
    print(hp.table("%s %s tangent" % (name, kw_id(kw)), e_ref["tangent"], e))
    check_bar(e, e_ref["tangent"], "%s %s tangent" % (name, kw_id(kw)))


# ---------------------------------------------------------------------------------------------------------------------
# Many right-hand sides
# ---------------------------------------------------------------------------------------------------------------------
# name: ((nx, nu, nc, nct, nc0, N), batch, mu, nrhs, right-hand sides measured (None: all))
MANY_CASES = {
    "c3_nrhs1": ((4, 2, 2, 2, 4, 5), 2, 1e-3, 1, None),
    "c3_nrhs17": ((4, 2, 2, 2, 4, 5), 2, 1e-3, 17, (0, 15, 16)),  # past the gradient kernel's 16-rhs chunk
    "c3_nrhs33": ((4, 2, 2, 2, 4, 5), 2, 1e-3, 33, (0, 15, 16, 31, 32)),  # past resolve's 32
    "rec510": ((11, 6, 4, 2, 11, 3), 1, 1e-3, 3, None),  # stage record just under the rho kernel's 512-double tile
    "rec518": ((12, 6, 1, 2, 12, 3), 1, 1e-3, 3, None),  # and just over it
    "c5_N1": ((57, 28, 0, 0, 57, 1), 1, 1e-2, 2, (0,)),     # the tiled 10 616-double record
}
MANY_ITEMS = [(n, kw) for n in MANY_CASES for kw in (DEFAULT, CTA) if not (n == "c5_N1" and kw is CTA)]


@functools.lru_cache(maxsize=None)
def many_cases(name):
    """One Case per right-hand side measured, sharing the problems; and all nrhs inputs."""
    d6, B, mu, nrhs, measured = MANY_CASES[name]
    probs = make_problems(d6, B, None, 7000 + sum(map(ord, name)))
    rng = np.random.default_rng(11)
    cots = [{k: rng.standard_normal(s) for k, s in aref._shapes(d6, B).items()} for _ in range(nrhs)]
    dots = [symmetric_dot(rng, d6, B) for _ in range(nrhs)]
    fcot = {k: None for k in ("ff", "fb", "vxx", "vx", "fft", "fbt")}
    if name == "c5_N1":
        fcot = c5_case().fcot
        cots[0], dots[0] = c5_case().cot, c5_case().dot
    js = range(nrhs) if measured is None else measured
    return probs, mu, cots, dots, {j: c5_case() if name == "c5_N1" and j == 0 else with_handle_dims(
        Case(probs, mu, inputs=dict(cot=cots[j], fcot=fcot, dot=dots[j])), d6) for j in js}


@functools.lru_cache(maxsize=None)
def c5_case():
    """C5 dims at horizon 1, one instance (extended precision at nx 57 is slow: one case serves both rows)."""
    d6, B, mu = MANY_CASES["c5_N1"][:3]
    return with_handle_dims(Case(make_problems(d6, B, None, 7000 + sum(map(ord, "c5_N1"))), mu), d6)


@pytest.mark.parametrize("name,kw", MANY_ITEMS, ids=["%s-%s" % (n, kw_id(kw)) for n, kw in MANY_ITEMS])
def test_many_rhs_meet_the_bar(env, name, kw):
    gar, _, torch = env
    probs, mu, cots, dots, cases = many_cases(name)
    c0 = next(iter(cases.values()))
    nrhs = len(cots)
    if name.startswith("rec"):
        nx, nu, nc = c0.d6[:3]
        assert gar.stage_record_doubles(nx, nu, nc) == int(name[3:])
    s = _handle(env, c0, kw)
    primal = {k: v.clone() for k, v in lq_gpu.primal(env, s).items()}
    stack = lambda ds: {k: _dev(torch, np.stack([d[k] for d in ds])) for k in ds[0]}
    nan = lambda shape: torch.full(shape, float("nan"), dtype=torch.float64, device="cuda")
    work = {k: nan((nrhs,) + tuple(v.shape)) for k, v in primal.items()}
    grad = {k: nan((nrhs,) + tuple(v.shape)) for k, v in lq_gpu.grad_bufs(env, s).items()}
    s.adjoint_many(primal, stack(cots), work, grad, mu)
    twork = {k: nan((nrhs,) + tuple(v.shape)) for k, v in primal.items()}
    out = {k: nan((nrhs,) + tuple(v.shape)) for k, v in primal.items()}
    s.tangent_many(primal, stack(dots), twork, out, mu)
    s.synchronize()
    G, Z = lq_gpu.to_np(grad), lq_gpu.to_np(out)
    s.close()
    for j, c in cases.items():
        e_ref = c.e_refs()
        e = c.e_adjoint({k: v[j] for k, v in G.items()})
        print("\n" + hp.table("%s %s adjoint_many rhs %d" % (name, kw_id(kw), j), e_ref["adjoint"], e))
        check_bar(e, e_ref["adjoint"], "%s %s adjoint_many rhs %d" % (name, kw_id(kw), j))
        e = c.e_tangent({k: v[j] for k, v in Z.items()})
        check_bar(e, e_ref["tangent"], "%s %s tangent_many rhs %d" % (name, kw_id(kw), j))


# ---------------------------------------------------------------------------------------------------------------------
# Derivatives of the factorisation
# ---------------------------------------------------------------------------------------------------------------------
def run_factor(env, c, kw, recs=None):
    """(factor_adjoint gradient, factor_tangent) of one handle after a backward on the case's problem."""
    gar, _, torch = env
    d6 = c.d6
    s = gar.CudaRiccatiBatch(*c.hdims, len(c.probs), **kw)
    s.set_problem(*[np.ascontiguousarray(a) for a in c.recs])
    s.backward(_mu_arg(torch, c.mu))
    assert np.all(s.status() == 0)
    g = lq_gpu.device_factor_adjoint(env, s, c.fcot, c.mu, d6)
    t = lq_gpu.device_factor_tangent(env, s, dict(stage=c.dot["stage"], term=c.dot["term"]), c.mu, d6)
    s.close()
    return g, t


def check_factor(c, g, t, title):
    e_ref, e_torch = c.e_refs(), c.e_torch()
    assert np.isfinite(g["stage"]).all() and not g["G0"].any() and not g["g0"].any(), title
    e = c.e_factor_adjoint(g)
    print("\n" + hp.table(title + " factor_adjoint", e_ref["factor_adjoint"], e, e_torch["factor_adjoint"]))
    check_bar(e, e_ref["factor_adjoint"], title + " factor_adjoint", e_torch["factor_adjoint"])
    e = c.e_factor_tangent(t)
    print(hp.table(title + " factor_tangent", e_ref["factor_tangent"], e, e_torch["factor_tangent"]))
    check_bar(e, e_ref["factor_tangent"], title + " factor_tangent", e_torch["factor_tangent"])


FACTOR_ITEMS = [(n, kw) for n in FACTOR_CASES for kw in ((DEFAULT,) if n in ("N0", "N1") else (DEFAULT, CTA))]


@pytest.mark.parametrize("name,kw", FACTOR_ITEMS, ids=["%s-%s" % (n, kw_id(kw)) for n, kw in FACTOR_ITEMS])
def test_factor_derivatives_meet_the_bar(env, name, kw):
    c = factor_case(name)
    g, t = run_factor(env, c, kw)
    check_factor(c, g, t, "%s %s" % (name, kw_id(kw)))


def test_factor_derivatives_c5_on_a_cta(env):
    """C5 dims at horizon 1, one instance: the 256-thread CTA item."""
    c = c5_case()
    g, t = run_factor(env, c, DEFAULT)
    check_factor(c, g, t, "c5_N1")


def problems_from_records(stage, term, G0, g0, d6):
    """Packed records -> LqrProblem list (the inverse of hp_reference.records)."""
    nx, nu, nc, nct, nc0, N = d6
    so, _ = aref.stage_offsets(nx, nu, nc)
    to, _ = aref.term_offsets(nx, nct)
    probs = []
    for b in range(term.shape[0]):
        knots = []
        for t in range(N + 1):
            k = LqrKnot(nx, nu, nc) if t < N else LqrKnot(nx, 0, nct)
            rec, off = (stage[b, t], so) if t < N else (term[b], to)
            for name, (a, e) in off.items():
                v = getattr(k, name)
                v[...] = rec[a:e].reshape(v.shape[::-1]).T if v.ndim == 2 else rec[a:e]
            knots.append(k)
        p = LqrProblem(knots, nc0)
        p.G0 = np.asfortranarray(G0[b].reshape(nx, nc0).T)
        p.g0 = np.array(g0[b], dtype=np.float64)
        probs.append(p)
    return probs


def test_factor_derivatives_after_cycle_append(env):
    """cycle_append, then a backward: the records are read through the ring head; the reference is the rotated
    problem."""
    gar, _, torch = env
    c = factor_case("c3_nct2_mu1e-3")
    d6, B = c.d6, len(c.probs)
    nx, nu, nc, nct, nc0, N = d6
    s = gar.CudaRiccatiBatch(*d6, B)
    s.set_problem(*[np.ascontiguousarray(a) for a in c.recs])
    s.backward(c.mu)
    new = make_problems((nx, nu, nc, nct, nc0, 1), B, None, 6200)
    _, srec = aref.stage_offsets(nx, nu, nc)
    nl = np.stack([np.pad(gen.stage_record(p.stages[0]), (0, srec - gen.stage_record(p.stages[0]).size))
                   for p in new])
    s.cycle_append(np.ascontiguousarray(nl))
    s.backward(c.mu)
    recs = (s.get_problem(0).reshape(B, N, -1), s.get_problem(1).reshape(B, -1), c.recs[2], c.recs[3])
    rotated = Case(problems_from_records(*recs, d6), c.mu, inputs=dict(cot=c.cot, fcot=c.fcot, dot=c.dot))
    rotated.hdims = d6
    assert np.array_equal(rotated.recs[0], recs[0]) and np.array_equal(rotated.recs[1], recs[1])
    g = lq_gpu.device_factor_adjoint(env, s, c.fcot, c.mu, d6)
    t = lq_gpu.device_factor_tangent(env, s, dict(stage=c.dot["stage"], term=c.dot["term"]), c.mu, d6)
    s.close()
    check_factor(rotated, g, t, "cycle_append")


# ---------------------------------------------------------------------------------------------------------------------
# Launch geometry: full-size batch counts, instances sampled across the launch
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [("C2", 12, 6, 0, 0, 4096, 1e-8, [0, 1, 263, 264, 2047, 2048, 4094, 4095]),
                                 ("C3", 4, 2, 2, 2, 16384, 1e-3, [0, 1, 511, 512, 8191, 8192, 16382, 16383])],
                         ids=["C2", "C3"])
def test_full_size_sampled_instances(env, cfg):
    gar, _, torch = env
    import bench
    name, nx, nu, nc, nct, B, mu, idx = cfg
    N = 10
    d6 = (nx, nu, nc, nct, nx, N)
    stage, term, G0, g0 = bench.synth_batch_torch(torch, B, N, nx, nu, "cuda:0", 78, nc, nct, "control")
    # Q, R and the terminal Q exactly symmetric from their lower triangles: one symmetric LQ problem whatever
    # rounding built them
    so, srec = aref.stage_offsets(nx, nu, nc)
    to, _ = aref.term_offsets(nx, nct)
    st = stage.view(B, N, -1)
    for x, off, k in ((st, so["Q"], nx), (st, so["R"], nu), (term, to["Q"], nx)):
        M = x[..., off[0]:off[1]].reshape(*x.shape[:-1], k, k)
        x[..., off[0]:off[1]] = (M.tril() + M.tril(-1).transpose(-1, -2)).reshape(*x.shape[:-1], k * k)
    recs = [a.cpu().numpy() for a in (stage.view(B, N, -1), term, G0, g0)]
    rng = np.random.default_rng(12)
    cot = {k: rng.standard_normal(sh) for k, sh in aref._shapes(d6, B).items()}
    fcot = {k: rng.standard_normal(sh) for k, sh in fadj.cot_shapes(d6, B).items()}
    dot = symmetric_dot(rng, d6, B)
    s = gar.CudaRiccatiBatch(*d6, B)
    s.set_problem(stage, term, G0, g0, memspace=gar.AB2_DEVICE)
    s.sweep(mu)
    assert np.all(s.status() == 0)
    primal = {k: v.clone() for k, v in lq_gpu.primal(env, s).items()}
    g = lq_gpu.grad_bufs(env, s)
    s.adjoint(primal, {k: _dev(torch, v) for k, v in cot.items()}, g, mu)
    s.synchronize()
    g = lq_gpu.to_np(g)
    s.tangent(primal, {k: _dev(torch, v) for k, v in dot.items()}, mu)
    s.synchronize()
    zd = lq_gpu.to_np(lq_gpu.primal(env, s))
    s.backward(mu)
    gf = lq_gpu.device_factor_adjoint(env, s, fcot, mu, d6)
    ft = lq_gpu.device_factor_tangent(env, s, dict(stage=dot["stage"], term=dot["term"]), mu, d6)
    s.close()
    pick = lambda d: {k: np.asarray(v)[idx] for k, v in d.items()}
    c = Case(problems_from_records(*[a[idx] for a in recs], d6), mu,
             inputs=dict(cot=pick(cot), fcot=pick(fcot), dot=pick(dot)))
    assert all(np.array_equal(a, b[idx]) for a, b in zip(c.recs, recs))
    e_ref = c.e_refs()
    e = c.e_adjoint(pick(g))
    print("\n" + hp.table("%s full size adjoint" % name, e_ref["adjoint"], e))
    check_bar(e, e_ref["adjoint"], "%s full size adjoint" % name)
    check_bar(c.e_tangent(pick(zd)), e_ref["tangent"], "%s full size tangent" % name)
    check_factor(c, pick(gf), pick(ft), "%s full size" % name)
