"""Jacobians of the LQ solve on the CPU (ab2_gar_adjoint_many / ab2_gar_tangent_many, gar.h): the batched formulas,
resolve then y z^T in reverse mode and resolve(rho) in forward mode, restated in numpy on top of the oracle's solve of
the replaced problem, against the single-cotangent adjoint and tangent references, and duality between the two for
every pair of right-hand sides.  Also the torch.func plumbing of autograd.lq_solve (vmap rules, broadcast of unbatched
cotangents, one device call per vmapped backward or jvp, vmap over the data refused), run against a linear stand-in
for the handle."""
import types

import numpy as np
import pytest

import gen
import lq_adjoint_ref as aref
import lq_resolve_ref as rref
import lq_tangent_ref as tref
from oracle import gar_oracle as orc

MU = 1e-2
# (nx, nu, nc, nct, nc0, N, B)
CASES = [(3, 2, 1, 1, 3, 4, 2), (4, 2, 1, 0, 0, 4, 1), (4, 3, 0, 1, 4, 0, 2), (5, 2, 1, 1, 1, 3, 2),
         (4, 2, 0, 1, 1, 1, 3)]
IDS = ["nx%d_nu%d_nc%d_nct%d_nc0%d_N%d_B%d" % c for c in CASES]
NRHS = 3


def _records(case, seed):
    nx, nu, nc, nct, nc0, N, B = case
    probs = gen.general_initial_condition(gen.generate_batch(seed, B, N, nx, nu, nc, nct), nc0, seed)
    _, srec = aref.stage_offsets(nx, nu, nc)
    stage = np.zeros((B, N, srec))
    for b, p in enumerate(probs):
        for t in range(N):
            r = gen.stage_record(p.stages[t])
            stage[b, t, :r.size] = r
    term = np.stack([gen.term_record(p.stages[N]) for p in probs])
    G0 = np.stack([np.asarray(p.G0).ravel(order="F") for p in probs]).reshape(B, nc0 * nx)
    g0 = np.stack([np.asarray(p.g0) for p in probs]).reshape(B, nc0)
    return stage, term, G0, g0


def _solve(case, recs):
    nx, nu, nc, nct, nc0, N, B = case
    bo = orc.BatchedOracle(nx, nu, nc, nct, nc0, N, B, *[np.ascontiguousarray(a) for a in recs])
    bo.sweep(MU, nthreads=1)
    assert np.all(bo.status == 1)  # the oracle reports 1 = ok
    return aref.oracle_dict(bo.get())


def _resolve(case, recs, h):
    """resolve(h) = -K^-1 h for ONE right-hand side: the oracle's solve of the problem with its vectors replaced."""
    return _solve(case, rref.replaced_records(*recs, h, case[:6]))


def grad_many(z, y, d6):
    """Gradient records from z and y = resolve(zbar) (the kernel's formulas: dh = y, dK = y z^T, symmetric part of
    Q and R)."""
    nx, nu, nc, nct, nc0, N = d6
    so, srec = aref.stage_offsets(nx, nu, nc)
    to, trec = aref.term_offsets(nx, nct)
    B = z["xs"].shape[0]
    o, cm = aref._outer, aref._cm
    pair = lambda a, b, ya, yb: o(ya, b) + o(a, yb)  # y_a b^T + a y_b^T
    x, u, v, l = z["xs"][:, :N], z["us"], z["vs"], z["lams"]
    X, U, V, L = y["xs"][:, :N], y["us"], y["vs"], y["lams"]
    blocks = dict(A=cm(pair(l, x, L, X)), B=cm(pair(l, u, L, U)), f=L, Q=cm(0.5 * pair(x, x, X, X)),
                  S=cm(pair(x, u, X, U)), R=cm(0.5 * pair(u, u, U, U)), q=X, r=U, C=cm(pair(v, x, V, X)),
                  D=cm(pair(v, u, V, U)), d=V)
    st = np.zeros((B, N, srec))
    for k, (a, b) in so.items():
        st[..., a:b] = blocks[k]
    xN, XN = z["xs"][:, N], y["xs"][:, N]
    tb = dict(Q=cm(0.5 * pair(xN, xN, XN, XN)), q=XN, C=cm(pair(z["vsT"], xN, y["vsT"], XN)), d=y["vsT"])
    tt = np.zeros((B, trec))
    for k, (a, b) in to.items():
        tt[:, a:b] = tb[k]
    G0 = cm(pair(z["lam0"], z["xs"][:, 0], y["lam0"], y["xs"][:, 0]))
    return dict(stage=st, term=tt, G0=G0, g0=y["lam0"])


def _cot_rhs(c):
    """A cotangent as resolve's right-hand side: xs -> q, us -> r, vs -> d, vsT -> dN, lam0 -> g0, lams -> f."""
    return dict(q=c["xs"], r=c["us"], d=c["vs"], dN=c["vsT"], g0=c["lam0"], f=c["lams"])


def _random(case, seed):
    nx, nu, nc, nct, nc0, N, B = case
    rng = np.random.default_rng(seed)
    _, srec = aref.stage_offsets(nx, nu, nc)
    _, trec = aref.term_offsets(nx, nct)
    cots = [{k: rng.standard_normal(s) for k, s in aref._shapes(case[:6], B).items()} for _ in range(NRHS)]
    dots = [dict(stage=rng.standard_normal((B, N, srec)), term=rng.standard_normal((B, trec)),
                 G0=rng.standard_normal((B, nc0 * nx)), g0=rng.standard_normal((B, nc0))) for _ in range(NRHS)]
    return cots, dots


def _rel(a, b):
    return max(gen.rel_fro(np.asarray(a[k]), np.asarray(b[k])) for k in b if np.asarray(b[k]).size)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_reverse_and_forward_formulas_match_single_references(case):
    d6 = case[:6]
    recs = _records(case, 5)
    z = _solve(case, recs)
    cots, dots = _random(case, 6)
    for j in range(NRHS):
        # reverse: y = resolve(zbar), then y z^T, against the adjoint reference (w = K^-1 zbar, dK = -w z^T)
        y = _resolve(case, recs, _cot_rhs(cots[j]))
        w = _solve(case, aref.adjoint_records(*recs, cots[j], d6))
        assert _rel(grad_many(z, y, d6), aref.grad_records(z, w, d6)) <= 1e-12, j
        # forward: resolve(rho), against the tangent reference (the tangent problem's solve)
        rho = tref.rho(dots[j], z, d6)
        zd = _resolve(case, recs, _cot_rhs(rho))
        assert _rel(zd, _solve(case, tref.tangent_records(*recs, dots[j], z, d6))) <= 1e-12, j


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_duality_for_every_pair(case):
    """<zbar_i, zdot_j> = <grad_i, pdot_j> for every (i, j), asymmetric Q and R tangents included."""
    d6 = case[:6]
    recs = _records(case, 8)
    z = _solve(case, recs)
    cots, dots = _random(case, 9)
    grads = [grad_many(z, _resolve(case, recs, _cot_rhs(c)), d6) for c in cots]
    zdots = [_resolve(case, recs, _cot_rhs(tref.rho(p, z, d6))) for p in dots]
    for i in range(NRHS):
        for j in range(NRHS):
            lhs = [cots[i][k] * zdots[j][k] for k in aref.KEYS]
            rhs = [grads[i][k] * dots[j][k] for k in ("stage", "term", "G0", "g0")]
            scale = max(sum(np.abs(a).sum() for a in lhs), sum(np.abs(a).sum() for a in rhs))
            assert abs(sum(a.sum() for a in lhs) - sum(a.sum() for a in rhs)) <= 1e-12 * scale, (i, j)


# ---- torch.func plumbing, against a linear stand-in for the handle ----
class _Linear:
    """A CudaRiccatiBatch stand-in whose 'solve' is z = M p (p the records): adjoint is M^T zbar, tangent M pdot, and
    the *_many calls do the same per right-hand side.  Counts the calls."""

    def __init__(self, torch, dense):
        self.torch, self.dense = torch, dense
        B, N, nx, nu, nc, nct, nc0 = 2, 3, 2, 1, 1, 1, 2
        self.dims = types.SimpleNamespace(batch=B, horizon=N, nx=nx, nu=nu, nc=nc, nct=nct, nc0=nc0)
        self.srec, self.trec = aref.stage_offsets(nx, nu, nc)[1], aref.term_offsets(nx, nct)[1]
        self.ins = dict(stage=(B, N, self.srec), term=(B, self.trec), G0=(B, nc0 * nx), g0=(B, nc0))
        self.outs = aref._shapes((nx, nu, nc, nct, nc0, N), B)
        n = lambda d: sum(int(np.prod(s)) for s in d.values())
        g = torch.Generator().manual_seed(0)
        self.M = torch.randn(n(self.outs), n(self.ins), generator=g, dtype=torch.float64)
        self.calls = {}

    def _count(self, k):
        self.calls[k] = self.calls.get(k, 0) + 1

    def _cat(self, d, shapes, j=None):
        z = self.torch.zeros
        return self.torch.cat([(z(s, dtype=self.torch.float64) if d.get(k) is None else
                                (d[k] if j is None else d[k][j])).reshape(-1) for k, s in shapes.items()])

    def _split(self, v, shapes):
        out, o = {}, 0
        for k, s in shapes.items():
            n = int(np.prod(s))
            out[k] = v[o:o + n].reshape(s)
            o += n
        return out

    def out_shape(self, w):
        return list(self.outs.values())[w - _gar().OUT_XS]

    def set_problem(self, stage, term, G0, g0, memspace=None, stream=0):
        self.p = self._cat(dict(stage=stage, term=term, G0=G0, g0=g0), self.ins)

    def sweep(self, mueq, stream=0):
        self.z = self._split(self.M @ self.p, self.outs)

    def backward(self, mueq, stream=0):
        pass

    def get_into(self, w, t, memspace, stream=0):
        t.copy_(self.z[list(self.outs)[w - _gar().OUT_XS]])

    def adjoint(self, primal, cot, grad, mueq, stream=0):
        self._count("adjoint")
        g = self._split(self.M.T @ self._cat(cot, self.outs), self.ins)
        for k, t in grad.items():
            t.copy_(g[k])

    def tangent(self, primal, dot, mueq, stream=0):
        self._count("tangent")
        self.z = self._split(self.M @ self._cat(dot, self.ins), self.outs)

    def adjoint_many(self, primal, cot, work, grad, mueq, stream=0):
        self._count("adjoint_many")
        for j in range(work["xs"].shape[0]):
            g = self._split(self.M.T @ self._cat(cot, self.outs, j), self.ins)
            for k, t in grad.items():
                t[j].copy_(g[k])

    def tangent_many(self, primal, dot, work, out, mueq, stream=0):
        self._count("tangent_many")
        for j in range(out["xs"].shape[0]):
            z = self._split(self.M @ self._cat(dot, self.ins, j), self.outs)
            for k, t in out.items():
                t[j].copy_(z[k])


def _gar():
    import aligator_b200.gar as gar
    return gar


@pytest.mark.parametrize("dense", [False, True], ids=["serial", "dense"])
def test_torch_func_plumbing(monkeypatch, dense):
    torch = pytest.importorskip("torch")
    import aligator_b200.autograd as ag
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: types.SimpleNamespace(cuda_stream=0))
    s = _Linear(torch, dense)
    g = torch.Generator().manual_seed(1)
    data = {k: torch.randn(sh, generator=g, dtype=torch.float64) for k, sh in s.ins.items()}
    solve = lambda st, tt, G0, g0: ag._LqSolve.apply(s, st, tt, G0, g0, MU)
    sizes = [int(np.prod(v)) for v in s.outs.values()]
    ni = int(np.prod(s.ins["stage"]))
    for k in (0, 1, 5):
        f = lambda st: solve(st, data["term"], data["G0"], data["g0"])[k]
        want = s.M[sum(sizes[:k]):sum(sizes[:k + 1]), :ni].reshape(tuple(s.outs.values())[k] + s.ins["stage"])
        s.calls.clear()
        Jr = torch.func.jacrev(f)(data["stage"])
        assert s.calls == ({"adjoint": sizes[k]} if dense else {"adjoint_many": 1}), s.calls
        s.calls.clear()
        Jf = torch.func.jacfwd(f)(data["stage"])
        assert s.calls == ({"tangent": ni} if dense else {"tangent_many": 1}), s.calls
        assert torch.equal(Jr, want) and torch.allclose(Jf, want, rtol=1e-14, atol=1e-14)
    # vmap of a vjp function with the cotangents batched along dimension 1; an unbatched cotangent is broadcast
    _, vjp_fn = torch.func.vjp(lambda st, g0: solve(st, data["term"], data["G0"], g0)[0], data["stage"], data["g0"])
    cots = torch.randn((s.dims.batch, 3) + tuple(s.outs["xs"][1:]), generator=g, dtype=torch.float64)
    gs = torch.func.vmap(vjp_fn, in_dims=1)(cots)
    for j in range(3):
        for a, b in zip(gs, vjp_fn(cots[:, j])):
            assert torch.allclose(a[j], b, rtol=1e-14, atol=1e-14)
    _, vjp2 = torch.func.vjp(lambda st: solve(st, data["term"], data["G0"], data["g0"])[:2], data["stage"])
    us = torch.randn(s.outs["us"], generator=g, dtype=torch.float64)
    gb = torch.func.vmap(vjp2, in_dims=((1, None),))((cots, us))[0]
    for j in range(3):
        assert torch.allclose(gb[j], vjp2((cots[:, j], us))[0], rtol=1e-14, atol=1e-14)
    # vmap over torch.func.jvp tangents
    tans = torch.randn((4,) + s.ins["term"], generator=g, dtype=torch.float64)
    h = lambda tt: solve(data["stage"], tt, data["G0"], data["g0"])
    jv = torch.func.vmap(lambda t: torch.func.jvp(h, (data["term"],), (t,))[1])(tans)
    for j in range(4):
        for a, b in zip(jv, torch.func.jvp(h, (data["term"],), (tans[j],))[1]):
            assert torch.allclose(a[j], b, rtol=1e-14, atol=1e-14)
    # vmap over the problem data is refused
    with pytest.raises(NotImplementedError, match="cotangents and tangents"):
        torch.func.vmap(lambda st: solve(st, data["term"], data["G0"], data["g0"]))(data["stage"].expand(2, -1, -1, -1))
    # not twice differentiable
    st = data["stage"].clone().requires_grad_(True)
    gst, = torch.autograd.grad(solve(st, data["term"], data["G0"], data["g0"])[0].sum(), st, create_graph=True)
    with pytest.raises(RuntimeError, match="differentiable once"):
        gst.sum().backward()


def test_lq_solve_argument_checks_without_a_gpu():
    torch = pytest.importorskip("torch")
    import aligator_b200.autograd as ag
    s = _Linear(torch, False)
    with pytest.raises(ValueError, match="CudaRiccatiBatch"):
        torch.func.jacrev(lambda st: ag.lq_solve(s, st, None, None, None, MU)[0])(torch.zeros(s.ins["stage"]))
    assert ag._LqSolve.vmap is not torch.autograd.Function.vmap
    with pytest.raises(NotImplementedError, match="cotangents and tangents"):
        ag._LqSolve.vmap(None, (None, 0, None, None, None, None), s, None, None, None, None, MU)
