"""Jacobians of the LQ solve on the GPU: many cotangents (ab2_gar_adjoint_many) and many tangents
(ab2_gar_tangent_many) on one factorisation, and jacrev / jacfwd / vmap of aligator_b200.autograd.lq_solve.  Parity with
separate ab2_gar_adjoint / ab2_gar_tangent calls and with the oracle, for every non-dense handle kind of the adjoint
tests; bit-exact independence of nrhs; NULL fields; the handle's outputs untouched; duality on the device; the
per-instance-mu twins; cycle_append; errors; torch.func; full-size configurations."""
import ctypes as C

import numpy as np
import pytest

import gen
import lq_adjoint_ref as aref
import lq_tangent_ref as tref
from oracle import gar_oracle as orc
from test_gpu_adjoint import HANDLES, MUS, _outputs, _primal, _setup, env  # noqa: F401  (env is the module fixture)
from test_gpu_resolve import SERIAL

pytestmark = pytest.mark.gpu
TOL = 1e-10
KEYS = aref.KEYS
RECS = ("stage", "term", "G0", "g0")


def _rec_shapes(s):
    d = s.dims
    return dict(stage=(d.batch, d.horizon, s.srec), term=(d.batch, s.trec), G0=(d.batch, d.nc0 * d.nx),
                g0=(d.batch, d.nc0))


def _randn(torch, shape, seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return torch.randn(shape, generator=g, dtype=torch.float64, device="cuda")


def _cots(env, s, primal, nrhs, seed):
    return {k: _randn(env[2], (nrhs,) + tuple(v.shape), seed + i) for i, (k, v) in enumerate(primal.items())}


def _dots(env, s, nrhs, seed):
    return {k: _randn(env[2], (nrhs,) + sh, seed + i) for i, (k, sh) in enumerate(_rec_shapes(s).items())}


def _nan(torch, shape):
    return torch.full(shape, float("nan"), dtype=torch.float64, device="cuda")


def _sol_bufs(env, primal, nrhs):
    return {k: _nan(env[2], (nrhs,) + tuple(v.shape)) for k, v in primal.items()}


def _grad_bufs(env, s, nrhs):
    return {k: _nan(env[2], (nrhs,) + sh) for k, sh in _rec_shapes(s).items()}


def _trajectory(env, s):
    gar = env[0]
    return {k: s.get(w) for k, w in zip(KEYS, (gar.OUT_XS, gar.OUT_US, gar.OUT_VS, gar.OUT_VST, gar.OUT_LBD0,
                                               gar.OUT_LBDAS))}


def _np(d):
    return {k: v.cpu().numpy() for k, v in d.items()}


def _oracle(dims, recs, mu):
    nx, nu, nc, nct, nc0, N, B = dims
    bo = orc.BatchedOracle(nx, nu, nc, nct, nc0, N, B, *[np.ascontiguousarray(a) for a in recs])
    bo.sweep(mu, nthreads=1)
    return aref.oracle_dict(bo.get())


def _tols(mu):
    # v_N = (d_N + C_N x_N) / mu: x_N's rounding error reaches the terminal multipliers (and the terminal gradient
    # record built from them) amplified by 1 / mu, as in test_gpu_resolve
    loose = max(TOL, 1e-13 / mu)
    return lambda k: loose if k in ("vsT", "term") else TOL


def _close(got, want, tol, tag):
    for k in want:
        if np.asarray(want[k]).size:
            e = gen.rel_fro(np.asarray(got[k]), np.asarray(want[k]))
            assert e <= tol(k), (tag, k, e)


@pytest.mark.parametrize("mu", MUS)
@pytest.mark.parametrize("name,kw,dims", SERIAL, ids=[h[0] for h in SERIAL])
def test_parity_with_single_calls_and_oracle(env, name, kw, dims, mu):
    gar, _, torch = env
    nx, nu, nc, nct, nc0, N, B = dims
    d6 = dims[:6]
    tol = _tols(mu)
    s, recs = _setup(env, kw, dims, 3, mu)
    primal = _primal(env, s)
    nrhs = 3
    cot, dot = _cots(env, s, primal, nrhs, 11), _dots(env, s, nrhs, 21)
    work, grad = _sol_bufs(env, primal, nrhs), _grad_bufs(env, s, nrhs)
    twork, out = _sol_bufs(env, primal, nrhs), _sol_bufs(env, primal, nrhs)
    before, e0 = _outputs(gar, s), s.factor_epoch()
    s.adjoint_many(primal, cot, work, grad, mu)
    s.tangent_many(primal, dot, twork, out, mu)
    s.synchronize()
    after = _outputs(gar, s)
    for k, a in before.items():  # every handle output is bit-equal before and after, and the epoch does not move
        assert np.array_equal(a, after[k], equal_nan=True), (name, k)
    assert s.factor_epoch() == e0
    G, Y, Z = _np(grad), _np(work), _np(out)
    assert np.all(G["stage"][..., aref.stage_offsets(nx, nu, nc)[0]["d"][1]:] == 0.0)  # the pad double
    zo = _oracle(dims, recs, mu)
    pn = _np(primal)
    for j in range(nrhs):
        cj = {k: v[j].cpu().numpy() for k, v in cot.items()}
        dj = {k: v[j].cpu().numpy() for k, v in dot.items()}
        # against the oracle: w = K^-1 zbar from the adjoint problem, zdot from the tangent problem
        w = _oracle(dims, aref.adjoint_records(*recs, cj, d6), mu)
        _close({k: v[j] for k, v in G.items()}, aref.grad_records(pn, w, d6), tol, (name, mu, j, "grad/oracle"))
        _close({k: v[j] for k, v in Y.items()}, {k: -v for k, v in w.items()}, tol, (name, mu, j, "y/oracle"))
        zd = _oracle(dims, tref.tangent_records(*recs, dj, zo, d6), mu)
        _close({k: v[j] for k, v in Z.items()}, zd, tol, (name, mu, j, "zdot/oracle"))
        # against separate single calls
        g1 = {k: torch.empty(sh, dtype=torch.float64, device="cuda") for k, sh in _rec_shapes(s).items()}
        s.adjoint(primal, {k: v[j] for k, v in cot.items()}, g1, mu)
        _close({k: v[j] for k, v in G.items()}, _np(g1), tol, (name, mu, j, "grad/adjoint"))
        s.tangent(primal, {k: v[j] for k, v in dot.items()}, mu)
        _close({k: v[j] for k, v in Z.items()}, _trajectory(env, s), tol, (name, mu, j, "zdot/tangent"))
    s.close()


@pytest.mark.parametrize("name,kw,dims", [SERIAL[i] for i in (0, 7, 9, 16, 17)],
                         ids=[SERIAL[i][0] for i in (0, 7, 9, 16, 17)])
def test_bits_null_fields_and_v_twins(env, name, kw, dims):
    gar, _, torch = env
    B = dims[-1]
    mu = 1e-2
    s, _ = _setup(env, kw, dims, 7, mu)
    primal = _primal(env, s)
    cot, dot = _cots(env, s, primal, 5, 31), _dots(env, s, 5, 41)
    work, grad = _sol_bufs(env, primal, 5), _grad_bufs(env, s, 5)
    twork, out = _sol_bufs(env, primal, 5), _sol_bufs(env, primal, 5)
    s.adjoint_many(primal, cot, work, grad, mu)
    s.tangent_many(primal, dot, twork, out, mu)
    # right-hand side j's results do not depend on nrhs or on j's position
    for j in (0, 2, 4):
        w1, g1 = _sol_bufs(env, primal, 1), _grad_bufs(env, s, 1)
        s.adjoint_many(primal, {k: v[j:j + 1].contiguous() for k, v in cot.items()}, w1, g1, mu)
        tw1, o1 = _sol_bufs(env, primal, 1), _sol_bufs(env, primal, 1)
        s.tangent_many(primal, {k: v[j:j + 1].contiguous() for k, v in dot.items()}, tw1, o1, mu)
        for k in RECS:
            assert torch.equal(g1[k][0], grad[k][j]), (name, j, k)
        for k in KEYS:
            assert torch.equal(w1[k][0], work[k][j]) and torch.equal(o1[k][0], out[k][j]), (name, j, k)
            assert torch.equal(tw1[k][0], twork[k][j]), (name, j, k)
    # NULL grad fields are not written; NULL cotangent and tangent fields are zeros
    part = {k: v[:2].contiguous() if k in ("xs", "lam0") else None for k, v in cot.items()}
    zeros = {k: v if v is not None else torch.zeros_like(cot[k][:2]) for k, v in part.items()}
    ga, gb = _grad_bufs(env, s, 2), _grad_bufs(env, s, 2)
    s.adjoint_many(primal, part, _sol_bufs(env, primal, 2), dict(stage=ga["stage"], g0=ga["g0"]), mu)
    s.adjoint_many(primal, zeros, _sol_bufs(env, primal, 2), gb, mu)
    assert torch.equal(ga["stage"], gb["stage"]) and torch.equal(ga["g0"], gb["g0"])
    assert torch.isnan(ga["term"]).all() and torch.isnan(ga["G0"]).all()
    tpart = {k: v[:2].contiguous() if k in ("term", "G0") else None for k, v in dot.items()}
    tzeros = {k: v if v is not None else torch.zeros_like(dot[k][:2]) for k, v in tpart.items()}
    oa, ob = _sol_bufs(env, primal, 2), _sol_bufs(env, primal, 2)
    s.tangent_many(primal, tpart, _sol_bufs(env, primal, 2), oa, mu)
    s.tangent_many(primal, tzeros, _sol_bufs(env, primal, 2), ob, mu)
    for k in KEYS:
        assert torch.equal(oa[k], ob[k]), (name, k)
    # the _v twins equal the scalar calls, with mu in host and in device memory
    for m in (np.full(B, mu), torch.full((B,), mu, dtype=torch.float64, device="cuda")):
        wv, gv = _sol_bufs(env, primal, 5), _grad_bufs(env, s, 5)
        s.adjoint_many(primal, cot, wv, gv, m)
        tv, ov = _sol_bufs(env, primal, 5), _sol_bufs(env, primal, 5)
        s.tangent_many(primal, dot, tv, ov, m)
        for k in RECS:
            assert torch.equal(gv[k], grad[k]), (name, k)
        for k in KEYS:
            assert torch.equal(wv[k], work[k]) and torch.equal(ov[k], out[k]), (name, k)
    s.close()


@pytest.mark.parametrize("name,kw,dims", [SERIAL[i] for i in (0, 7, 16, 17)],
                         ids=[SERIAL[i][0] for i in (0, 7, 16, 17)])
def test_duality_on_device(env, name, kw, dims):
    """<zbar_i, zdot_j> = <grad_i, pdot_j> for 3 x 3 pairs."""
    gar, _, torch = env
    mu = 1e-2
    s, _ = _setup(env, kw, dims, 9, mu)
    primal = _primal(env, s)
    cot, dot = _cots(env, s, primal, 3, 51), _dots(env, s, 3, 61)
    work, grad = _sol_bufs(env, primal, 3), _grad_bufs(env, s, 3)
    twork, out = _sol_bufs(env, primal, 3), _sol_bufs(env, primal, 3)
    s.adjoint_many(primal, cot, work, grad, mu)
    s.tangent_many(primal, dot, twork, out, mu)
    for i in range(3):
        for j in range(3):
            lhs = sum(float((cot[k][i] * out[k][j]).sum()) for k in KEYS)
            rhs = sum(float((grad[k][i] * dot[k][j]).sum()) for k in RECS)
            scale = max(sum(float((cot[k][i] * out[k][j]).abs().sum()) for k in KEYS),
                        sum(float((grad[k][i] * dot[k][j]).abs().sum()) for k in RECS))
            assert abs(lhs - rhs) <= 1e-12 * scale, (name, i, j, lhs, rhs)
    s.close()


def test_cycle_append(env):
    gar, _, torch = env
    dims = (4, 2, 2, 2, 4, 6, 9)
    nx, nu, nc, nct, nc0, N, B = dims
    mu = 1e-2
    s, _ = _setup(env, {}, dims, 1, mu)
    new_last = np.ascontiguousarray(gen.stage_record(gen.generate_batch(9, 1, 1, nx, nu, nc, nct)[0].stages[0]))
    nl = np.zeros((B, s.srec))
    nl[:, :new_last.size] = new_last
    s.cycle_append(nl)
    primal = _primal(env, s)
    cot, dot = _cots(env, s, primal, 2, 71), _dots(env, s, 2, 81)
    with pytest.raises(gar.GarError):  # no backward since cycle_append
        s.adjoint_many(primal, cot, _sol_bufs(env, primal, 2), _grad_bufs(env, s, 2), mu)
    s.sweep(mu)
    primal = _primal(env, s)
    work, grad = _sol_bufs(env, primal, 2), _grad_bufs(env, s, 2)
    twork, out = _sol_bufs(env, primal, 2), _sol_bufs(env, primal, 2)
    s.adjoint_many(primal, cot, work, grad, mu)
    s.tangent_many(primal, dot, twork, out, mu)
    for j in range(2):
        g1 = {k: torch.empty(sh, dtype=torch.float64, device="cuda") for k, sh in _rec_shapes(s).items()}
        s.adjoint(primal, {k: v[j] for k, v in cot.items()}, g1, mu)
        _close({k: v[j] for k, v in _np(grad).items()}, _np(g1), _tols(mu), j)
        s.tangent(primal, {k: v[j] for k, v in dot.items()}, mu)
        _close({k: v[j] for k, v in _np(out).items()}, _trajectory(env, s), _tols(mu), j)
    s.close()


def _rc_adj(gar, s, mu, nrhs, primal, cot, work, grad):
    f = lambda st, keys, d: gar._fill(st, keys, d)
    return gar.lib().ab2_gar_adjoint_many(s.h, C.c_double(mu), int(nrhs), C.byref(f(gar.LsIterate(), gar._LS_KEYS, primal)),
                                          C.byref(f(gar.LsIterate(), gar._LS_KEYS, cot)),
                                          C.byref(f(gar.LsIterate(), gar._LS_KEYS, work)),
                                          C.byref(f(gar.LqGrad(), gar._GRAD_KEYS, grad)), None)


def _rc_tan(gar, s, mu, nrhs, primal, dot, work, out):
    f = lambda st, keys, d: gar._fill(st, keys, d)
    return gar.lib().ab2_gar_tangent_many(s.h, C.c_double(mu), int(nrhs), C.byref(f(gar.LsIterate(), gar._LS_KEYS, primal)),
                                          C.byref(f(gar.LqTangent(), gar._GRAD_KEYS, dot)),
                                          C.byref(f(gar.LsIterate(), gar._LS_KEYS, work)),
                                          C.byref(f(gar.LsIterate(), gar._LS_KEYS, out)), None)


def test_state_and_errors(env):
    gar, _, torch = env
    dims = (4, 2, 2, 2, 4, 6, 9)
    nx, nu, nc, nct, nc0, N, B = dims
    mu = 1e-2
    probs = gen.generate_batch(1, B, N, nx, nu, nc, nct)
    recs = gar.pack_problems(probs)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    shapes = dict(xs=(B, N + 1, nx), us=(B, N, nu), vs=(B, N, nc), vsT=(B, nct), lam0=(B, nc0), lams=(B, N, nx))
    primal = {k: torch.zeros(sh, dtype=torch.float64, device="cuda") for k, sh in shapes.items()}
    cot = {k: torch.zeros((2,) + sh, dtype=torch.float64, device="cuda") for k, sh in shapes.items()}
    work = {k: torch.zeros((2,) + sh, dtype=torch.float64, device="cuda") for k, sh in shapes.items()}
    out = {k: torch.zeros((2,) + sh, dtype=torch.float64, device="cuda") for k, sh in shapes.items()}
    grad = {k: torch.zeros((2,) + sh, dtype=torch.float64, device="cuda") for k, sh in _rec_shapes(s).items()}
    dot = {k: torch.zeros((2,) + sh, dtype=torch.float64, device="cuda") for k, sh in _rec_shapes(s).items()}
    adj = lambda **kw: _rc_adj(gar, s, kw.get("mu", mu), kw.get("nrhs", 2), kw.get("primal", primal), kw.get("cot", cot),
                               kw.get("work", work), kw.get("grad", grad))
    tan = lambda **kw: _rc_tan(gar, s, kw.get("mu", mu), kw.get("nrhs", 2), kw.get("primal", primal), kw.get("dot", dot),
                               kw.get("work", work), kw.get("out", out))
    assert adj() == 4 and tan() == 4  # no problem
    s.set_problem(*recs)
    assert adj() == 4 and tan() == 4  # no backward since set_problem
    s.sweep(mu)
    s.synchronize()
    n0 = s.launch_count()
    for f in (adj, tan):
        assert f(nrhs=-1) == 1
        assert f(mu=0.0) == 1
        for k in KEYS:
            assert f(work=dict(work, **{k: None})) == 1, k
            assert f(primal=dict(primal, **{k: None})) == 1, k
        assert f(work=dict(work, us=primal["us"]), nrhs=1) == 1  # work overlaps primal
        assert f(nrhs=0) == 0
    for k in KEYS:
        assert tan(out=dict(out, **{k: None})) == 1, k
    # overlaps that would let a step read what an earlier step wrote
    assert adj(cot=dict(cot, vs=work["vs"])) == 1
    assert adj(grad=dict(grad, g0=primal["lam0"][:1].reshape(-1))) == 1
    assert adj(grad=dict(grad, G0=work["xs"].reshape(-1)[3:])) == 1
    assert adj(grad=dict(grad, g0=grad["stage"].reshape(-1)[5:])) == 1
    assert tan(dot=dict(dot, g0=work["lam0"])) == 1
    assert tan(out=dict(out, lams=work["lams"])) == 1
    assert tan(out=dict(out, xs=primal["xs"]), nrhs=1) == 1
    assert tan(out=dict(out, us=out["lams"].reshape(-1)[1:])) == 1
    s.synchronize()
    assert s.launch_count() == n0  # nothing launched on an error or for nrhs = 0
    assert adj() == 0 and s.launch_count() == n0 + 2
    assert tan() == 0 and s.launch_count() == n0 + 4
    s.close()
    for kw in (dict(dense=True), dict(legs=2), dict(nth=2)):
        u = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
        assert _rc_adj(gar, u, mu, 2, primal, cot, work, grad) == 2, kw
        assert _rc_tan(gar, u, mu, 2, primal, dot, work, out) == 2, kw
        u.close()


def _counting(s, name, calls):
    f = getattr(s, name)

    def wrapped(*a, **kw):
        calls[name] = calls.get(name, 0) + 1
        return f(*a, **kw)
    setattr(s, name, wrapped)


@pytest.mark.parametrize("dense", [False, True], ids=["serial", "dense"])
def test_torch_func(env, dense):
    gar, ag, torch = env
    dims = (4, 2, 2, 2, 4, 3, 2)
    nx, nu, nc, nct, nc0, N, B = dims
    mu = 1e-2
    s, recs = _setup(env, dict(dense=dense), dims, 13, mu)
    calls = {}
    for n in ("adjoint", "tangent", "adjoint_many", "tangent_many"):
        _counting(s, n, calls)
    stage, term, G0, g0 = [torch.tensor(np.ascontiguousarray(a), device="cuda").reshape(sh)
                           for a, sh in zip(recs, _rec_shapes(s).values())]
    for k in (0, 1, 5):  # xs, us, lams
        f = lambda st: ag.lq_solve(s, st, term, G0, g0, mu)[k]
        calls.clear()
        Jr = torch.func.jacrev(f)(stage)
        assert calls.get("adjoint_many", 0) == (0 if dense else 1), calls
        calls.clear()
        Jf = torch.func.jacfwd(f)(stage)
        assert calls.get("tangent_many", 0) == (0 if dense else 1), calls
        assert gen.rel_fro(Jr.cpu().numpy(), Jf.cpu().numpy()) <= TOL, k
        # rows from unbatched autograd.grad, columns from unbatched torch.func.jvp
        st = stage.clone().requires_grad_(True)
        y = ag.lq_solve(s, st, term, G0, g0, mu)[k]
        # relative to the whole Jacobian: some rows and columns are zero up to rounding (x_0 is pinned by nc0 = nx)
        flat, scale = Jr.reshape(y.numel(), -1), float(Jr.norm())
        for r in range(0, y.numel(), 7):
            e = torch.zeros(y.numel(), dtype=torch.float64, device="cuda")
            e[r] = 1.0
            row, = torch.autograd.grad(y, st, e.reshape(y.shape), retain_graph=True)
            assert float((flat[r] - row.reshape(-1)).norm()) <= TOL * scale, (k, r)
        flatf = Jf.reshape(y.numel(), -1)
        for c in range(0, stage.numel(), 37):
            e = torch.zeros(stage.numel(), dtype=torch.float64, device="cuda")
            e[c] = 1.0
            _, col = torch.func.jvp(f, (stage,), (e.reshape(stage.shape),))
            assert float((flatf[:, c] - col.reshape(-1)).norm()) <= TOL * scale, (k, c)
    # vmap of a vjp function with the cotangents batched along dimension 1
    out, vjp_fn = torch.func.vjp(lambda a, b: ag.lq_solve(s, a, term, G0, b, mu)[0], stage, g0)
    cots = torch.randn((B, 3) + tuple(out.shape[1:]), dtype=torch.float64, device="cuda")
    calls.clear()
    gs = torch.func.vmap(vjp_fn, in_dims=1)(cots)
    assert calls.get("adjoint_many", 0) == (0 if dense else 1), calls
    for j in range(3):
        g1 = vjp_fn(cots[:, j])
        for a, b in zip(gs, g1):
            assert gen.rel_fro(a[j].cpu().numpy(), b.cpu().numpy()) <= TOL, j
    # vmap over torch.func.jvp tangents of term and G0
    tans = (torch.randn((4,) + tuple(term.shape), dtype=torch.float64, device="cuda"),
            torch.randn((4,) + tuple(G0.shape), dtype=torch.float64, device="cuda"))
    h = lambda a, b: ag.lq_solve(s, stage, a, b, g0, mu)
    calls.clear()
    jv = torch.func.vmap(lambda ta, tb: torch.func.jvp(h, (term, G0), (ta, tb))[1])(*tans)
    assert calls.get("tangent_many", 0) == (0 if dense else 1), calls
    for j in range(4):
        one = torch.func.jvp(h, (term, G0), (tans[0][j], tans[1][j]))[1]
        for a, b in zip(jv, one):
            assert gen.rel_fro(a[j].cpu().numpy(), b.cpu().numpy()) <= TOL, j
    # vmap over the problem data is refused
    with pytest.raises(NotImplementedError, match="cotangents and tangents"):
        torch.func.vmap(lambda st: ag.lq_solve(s, st, term, G0, g0, mu)[0])(stage.unsqueeze(0).expand(2, -1, -1, -1)
                                                                              .contiguous())
    # outside vmap, gradients and jvps are bit-equal to direct adjoint and tangent calls
    leaves = [t.clone().requires_grad_(True) for t in (stage, term, G0, g0)]
    outs = ag.lq_solve(s, *leaves, mu)
    cot = {k: torch.randn_like(o) for k, o in zip(KEYS, outs)}
    got = torch.autograd.grad(outs, leaves, [cot[k] for k in KEYS])
    primal = {k: o.detach().clone() for k, o in zip(KEYS, outs)}
    want = {k: torch.empty_like(t) for k, t in zip(RECS, (stage, term, G0, g0))}
    s.set_problem(stage, term, G0, g0, memspace=gar.AB2_DEVICE)
    s.adjoint(primal, cot, want, mu)
    for k, a in zip(RECS, got):
        assert torch.equal(a, want[k]), k
    dots = tuple(torch.randn_like(t) for t in (stage, term, G0, g0))
    _, jo = torch.func.jvp(lambda *a: ag.lq_solve(s, *a, mu), (stage, term, G0, g0), dots)
    s.set_problem(stage, term, G0, g0, memspace=gar.AB2_DEVICE)
    s.tangent(primal, dict(zip(RECS, dots)), mu)
    for k, a in zip(KEYS, jo):
        assert np.array_equal(a.cpu().numpy(), _trajectory(env, s)[k]), k
    s.close()


@pytest.mark.parametrize("dims", [(12, 6, 0, 0, 12, 100, 4096), (4, 2, 2, 2, 4, 100, 16384)], ids=["C2", "C3"])
def test_full_size(env, dims):
    gar, _, torch = env
    nx, nu, nc, nct, nc0, N, B = dims
    mu = 1e-2
    nrhs = 4
    s, _ = _setup(env, {}, dims, 2, mu)
    primal = _primal(env, s)
    idx = torch.tensor(np.r_[0:3, B // 2 - 2:B // 2 + 2, B - 5:B], device="cuda")  # first wave, a wave boundary, the tail
    cot = _cots(env, s, primal, nrhs, 91)
    work, grad = _sol_bufs(env, primal, nrhs), _grad_bufs(env, s, nrhs)
    s.adjoint_many(primal, cot, work, grad, mu)
    sub = {k: v[:, idx].cpu().numpy() for k, v in grad.items()}
    del work, grad
    for j in (0, nrhs - 1):
        g1 = {k: torch.empty(sh, dtype=torch.float64, device="cuda") for k, sh in _rec_shapes(s).items()}
        s.adjoint(primal, {k: v[j] for k, v in cot.items()}, g1, mu)
        _close({k: v[j] for k, v in sub.items()}, {k: v[idx].cpu().numpy() for k, v in g1.items()}, _tols(mu), j)
        del g1
    del cot
    torch.cuda.empty_cache()
    dot = _dots(env, s, nrhs, 93)
    work, out = _sol_bufs(env, primal, nrhs), _sol_bufs(env, primal, nrhs)
    s.tangent_many(primal, dot, work, out, mu)
    for j in (0, nrhs - 1):
        s.tangent(primal, {k: v[j] for k, v in dot.items()}, mu)
        want = _trajectory(env, s)
        _close({k: v[j][idx].cpu().numpy() for k, v in out.items()}, {k: v[idx.cpu().numpy()] for k, v in want.items()},
               _tols(mu), j)
    s.close()
