"""Higher derivatives of the LQ solve on the CPU (ab2_gar_rho_many / ab2_gar_grad_many and lq_solve_higher, gar.h,
DESIGN section 2p).

* The two kernel modes restated in numpy (per-direction vectors, two terms, with and without the vector blocks, e), on
  top of lq_tangent_ref.rho and lq_higher_ref.grad_many, against a dense Kdot: K is affine in the data P, so
  Kdot = K(P + Pdot) - K(P) of the dense KKT matrix (gen.lqr_dense_kkt); and the pairing identities.
* The torch plumbing of lq_solve_higher against a CPU stand-in for the handle that solves the dense KKT systems in
  float64 and runs the numpy restatements for rho_many / grad_many, checked against a pure-torch differentiable dense
  solve: values, grad, grad of grad, hessian, jvp of grad, jacfwd(jacfwd), jacrev(jacfwd), a third derivative, the
  number of device calls under hessian, and the refusals.  Where a composition nests forward mode inside another
  transform, the reference is differentiated in reverse mode throughout: its own forward-over-forward and
  reverse-over-forward derivatives through torch.linalg.solve disagree with its reverse-mode ones."""
import types

import numpy as np
import pytest

import gen
import lq_adjoint_ref as aref
from lq_cases import jacobian_records
from lq_higher_ref import grad_modes, rho_modes

MU = 0.1
# (nx, nu, nc, nct, nc0, N, B)
CASES = [(3, 2, 1, 1, 3, 3, 2), (2, 1, 0, 1, 2, 2, 2), (3, 2, 1, 0, 1, 2, 1)]
IDS = ["nx%d_nu%d_nc%d_nct%d_nc0%d_N%d_B%d" % c for c in CASES]
KEYS = aref.KEYS
RECS = ("stage", "term", "G0", "g0")
HVP_CALLS = dict(backward=1, resolve=3, grad_many=2, rho_many=2)  # device calls of a hessian or a batch of HVPs


# ---- the dense KKT system of one instance, from the records ----
def _problem(stage, term, G0, g0, b, d6):
    """Instance b of the records as the problem object gen.lqr_dense_kkt reads, with Q and R taken through their
    symmetric part (the kernels' convention for Q and R)."""
    nx, nu, nc, nct, nc0, N = d6
    so, _ = aref.stage_offsets(nx, nu, nc)
    to, _ = aref.term_offsets(nx, nct)
    blk = lambda rec, off, m, n: np.asarray(rec[off[0]:off[1]]).reshape(n, m).T
    sym = lambda M: 0.5 * (M + M.T)
    knots = []
    for t in range(N):
        r = stage[b, t]
        knots.append(types.SimpleNamespace(
            nx=nx, nu=nu, nc=nc, nx2=nx, A=blk(r, so["A"], nx, nx), B=blk(r, so["B"], nx, nu),
            f=r[so["f"][0]:so["f"][1]],
            Q=sym(blk(r, so["Q"], nx, nx)), S=blk(r, so["S"], nx, nu), R=sym(blk(r, so["R"], nu, nu)),
            q=r[so["q"][0]:so["q"][1]], r=r[so["r"][0]:so["r"][1]], C=blk(r, so["C"], nc, nx),
            D=blk(r, so["D"], nc, nu), d=r[so["d"][0]:so["d"][1]]))
    r = term[b]
    knots.append(types.SimpleNamespace(
        nx=nx, nu=0, nc=nct, nx2=nx, Q=sym(blk(r, to["Q"], nx, nx)), S=np.zeros((nx, 0)), R=np.zeros((0, 0)),
        q=r[to["q"][0]:to["q"][1]], r=np.zeros(0), C=blk(r, to["C"], nct, nx), D=np.zeros((nct, 0)),
        d=r[to["d"][0]:to["d"][1]]))
    return types.SimpleNamespace(stages=knots, horizon=N, nc0=nc0, G0=np.asarray(G0[b]).reshape(nx, nc0).T,
                                 g0=np.asarray(g0[b]))


def dense_kkt(recs, b, d6, mu=MU):
    K, h, _ = gen.lqr_dense_kkt(_problem(*recs, b, d6), mu)
    return K, h


def _order(d6):
    """Index of every entry of the dense unknown [lam0, (x_t, u_t, v_t, lam_{t+1})_t, x_N, v_N] in the concatenation
    of one instance's solution fields (xs, us, vs, vsT, lam0, lams), each flattened."""
    nx, nu, nc, nct, nc0, N = d6
    sizes = [(N + 1) * nx, N * nu, N * nc, nct, nc0, N * nx]
    base = np.cumsum([0] + sizes)
    idx = list(base[4] + np.arange(nc0))
    for t in range(N):
        idx += list(base[0] + t * nx + np.arange(nx)) + list(base[1] + t * nu + np.arange(nu))
        idx += list(base[2] + t * nc + np.arange(nc)) + list(base[5] + t * nx + np.arange(nx))
    idx += list(base[0] + N * nx + np.arange(nx)) + list(base[3] + np.arange(nct))
    return np.array(idx, dtype=np.int64), sizes


def to_dense(v, b, d6):
    idx, _ = _order(d6)
    flat = np.concatenate([np.asarray(v[k][b]).ravel() for k in KEYS])
    return flat[idx]


def from_dense(x, d6, B=1):
    """Dense vectors x [B][n] -> solution dict [B][...]."""
    idx, sizes = _order(d6)
    flat = np.zeros((B, sum(sizes)))
    flat[:, idx] = x
    shapes = aref._shapes(d6, B)
    out, o = {}, 0
    for k, n in zip(KEYS, sizes):
        out[k] = flat[:, o:o + n].reshape(shapes[k])
        o += n
    return out


def _random_recs(case, rng, nrhs):
    nx, nu, nc, nct, nc0, N, B = case
    _, srec = aref.stage_offsets(nx, nu, nc)
    _, trec = aref.term_offsets(nx, nct)
    return dict(stage=rng.standard_normal((nrhs, B, N, srec)), term=rng.standard_normal((nrhs, B, trec)),
                G0=rng.standard_normal((nrhs, B, nc0 * nx)), g0=rng.standard_normal((nrhs, B, nc0)))


def _random_vec(case, rng, lead):
    return {k: rng.standard_normal(lead + s) for k, s in aref._shapes(case[:6], case[6]).items()}


def _pair(a, b):
    return sum(float(np.sum(a[k] * b[k])) for k in b)


def _scale(a, b):
    return sum(float(np.sum(np.abs(a[k] * b[k]))) for k in b)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_rho_modes_against_dense_kdot(case):
    d6, B, nrhs = case[:6], case[6], 3
    rng = np.random.default_rng(1)
    recs = jacobian_records(case, 3)
    dot1, dot2 = _random_recs(case, rng, nrhs), _random_recs(case, rng, nrhs)
    a1, a2, e = _random_vec(case, rng, (nrhs,)), _random_vec(case, rng, ()), _random_vec(case, rng, (nrhs,))
    a2["each"] = False
    for vec in (True, False):
        got = rho_modes(nrhs, d6, dot1, a1, vec, dot2, a2, e)
        for j in range(nrhs):
            for b in range(B):
                want = to_dense({k: e[k][j] for k in KEYS}, b, d6).copy()
                for P, a, v in ((dot1, {k: a1[k][j] for k in KEYS}, vec), (dot2, a2, False)):
                    Pd = {k: P[k][j] for k in RECS}
                    plus = [recs[i] + Pd[k] for i, k in enumerate(RECS)]
                    K0, h0 = dense_kkt(recs, b, d6)
                    K1, h1 = dense_kkt(plus, b, d6)
                    want += (K1 - K0) @ to_dense(a, b, d6) + (h1 - h0 if v else 0.0)
                r = to_dense({k: got[k][j] for k in KEYS}, b, d6)
                assert np.linalg.norm(r - want) <= 1e-12 * max(1.0, np.linalg.norm(want)), (vec, j, b)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_pairing_identities_and_symmetry(case):
    """<Gr(y; z), Pdot> = <y, rho(Pdot; z)>, <Gr_K(y; z), Pdot> = <y, rho_K(Pdot; z)> = <z, rho_K(Pdot; y)>, and
    Gr_K(y; z) = Gr_K(z; y); two terms are the sums of one-term calls."""
    d6, nrhs = case[:6], 4
    rng = np.random.default_rng(2)
    P = _random_recs(case, rng, nrhs)
    y, z, y2, z2 = (_random_vec(case, rng, (nrhs,)) for _ in range(4))
    for vec in (True, False):
        G = grad_modes(nrhs, d6, y, z, vec)
        R = rho_modes(nrhs, d6, P, z, vec)
        lhs, rhs = _pair(G, {k: P[k] for k in RECS}), _pair(y, R)
        assert abs(lhs - rhs) <= 1e-12 * _scale(y, R), vec
    GK = grad_modes(nrhs, d6, y, z, False)
    GKs = grad_modes(nrhs, d6, z, y, False)
    for k in RECS:
        assert np.allclose(GK[k], GKs[k], rtol=1e-12, atol=1e-12 * np.abs(GK[k]).max(initial=1.0)), k
    Rz = rho_modes(nrhs, d6, P, y, False)
    assert abs(_pair(z, Rz) - _pair(y, rho_modes(nrhs, d6, P, z, False))) <= 1e-12 * _scale(z, Rz)
    two = grad_modes(nrhs, d6, y, z, True, y2, z2)
    one = [grad_modes(nrhs, d6, y, z, True), grad_modes(nrhs, d6, y2, z2, False)]
    for k in RECS:
        assert np.allclose(two[k], one[0][k] + one[1][k], rtol=1e-13, atol=1e-13), k


# ---- torch plumbing of lq_solve_higher, against a dense CPU stand-in for the handle ----
class _DenseHandle:
    """A CudaRiccatiBatch stand-in: sweep, backward and resolve solve the dense KKT systems of the records (float64),
    rho_many and grad_many run the numpy restatements.  Counts the calls."""

    def __init__(self, torch, case):
        self.torch = torch
        nx, nu, nc, nct, nc0, N, B = case
        self.d6 = case[:6]
        self.dims = types.SimpleNamespace(batch=B, horizon=N, nx=nx, nu=nu, nc=nc, nct=nct, nc0=nc0, device=0)
        self.srec, self.trec = aref.stage_offsets(nx, nu, nc)[1], aref.term_offsets(nx, nct)[1]
        self.dense, self.nth, self.legs = False, 0, 0
        self.shapes = aref._shapes(self.d6, B)
        self.epoch, self.calls = 0, {}

    def _count(self, k):
        self.calls[k] = self.calls.get(k, 0) + 1

    def _np(self, d):
        return {k: None if v is None else v.detach().numpy() for k, v in d.items() if k != "each"}

    def out_shape(self, w):
        import aligator_b200.gar as gar
        return self.shapes[KEYS[w - gar.OUT_XS]]

    def set_problem(self, stage, term, G0, g0, memspace=None, stream=0):
        self.recs = [t.detach().numpy().copy() for t in (stage, term, G0, g0)]
        self.epoch += 1

    def backward(self, mueq, stream=0):
        self._count("backward")
        self.K = [dense_kkt(self.recs, b, self.d6, mueq) for b in range(self.dims.batch)]
        self.epoch += 1

    def sweep(self, mueq, stream=0):
        self.backward(mueq)
        self.z = from_dense(np.stack([np.linalg.solve(K, -h) for K, h in self.K]), self.d6, self.dims.batch)

    def get_into(self, w, t, memspace, stream=0):
        import aligator_b200.gar as gar
        t.copy_(self.torch.from_numpy(self.z[KEYS[w - gar.OUT_XS]]))

    def factor_epoch(self):
        return self.epoch

    def resolve(self, rhs, out, mueq, stream=0):
        self._count("resolve")
        nrhs, B = out["xs"].shape[0], self.dims.batch
        rhs = {k: None if rhs.get(r) is None else rhs[r].numpy().reshape((nrhs,) + self.shapes[k])
               for k, r in zip(KEYS, ("q", "r", "d", "dN", "g0", "f"))}
        for j in range(nrhs):
            h = aref._full({k: None if v is None else v[j] for k, v in rhs.items()}, self.d6, B)
            z = from_dense(np.stack([np.linalg.solve(self.K[b][0], -to_dense(h, b, self.d6)) for b in range(B)]),
                           self.d6, B)
            for k in KEYS:
                out[k][j].copy_(self.torch.from_numpy(z[k]))

    def _vec(self, v, nrhs):
        d = self._np(v)
        if d["xs"].shape == self.shapes["xs"]:
            d["each"] = False
        return d

    def rho_many(self, dot, a, out, vectors=True, dot2=None, a2=None, e=None, stream=0):
        self._count("rho_many")
        nrhs = out["xs"].shape[0]
        r = rho_modes(nrhs, self.d6, self._np(dot), self._vec(a, nrhs), vectors,
                      None if dot2 is None else self._np(dot2), None if a2 is None else self._vec(a2, nrhs),
                      None if e is None else self._np(e))
        for k in KEYS:
            out[k].copy_(self.torch.from_numpy(r[k]))

    def grad_many(self, y, z, grad, vectors=True, y2=None, z2=None, stream=0):
        self._count("grad_many")
        nrhs = y["xs"].shape[0]
        g = grad_modes(nrhs, self.d6, self._np(y), self._vec(z, nrhs), vectors,
                       None if y2 is None else self._np(y2), None if z2 is None else self._vec(z2, nrhs))
        for k, t in grad.items():
            t.copy_(self.torch.from_numpy(g[k]))


def _torch_reference(torch, case, recs):
    """A pure-torch differentiable dense KKT solve: K(p) and h(p) are affine in the records p, so they are the torch
    maps K(0) + dK p, dh p with the columns of dK and dh read off gen.lqr_dense_kkt at unit records."""
    nx, nu, nc, nct, nc0, N, B = case
    d6 = case[:6]
    sizes = [int(np.prod(r.shape[1:])) for r in recs]
    n_p = sum(sizes)

    def unflat(p):
        out, o = [], 0
        for r, n in zip(recs, sizes):
            out.append(p[o:o + n].reshape((1,) + r.shape[1:]))
            o += n
        return out

    K0, h0 = dense_kkt(unflat(np.zeros(n_p)), 0, d6)
    cols = [dense_kkt(unflat(np.eye(n_p)[i]), 0, d6) for i in range(n_p)]
    dK = torch.from_numpy(np.stack([K - K0 for K, _ in cols], axis=-1))
    dh = torch.from_numpy(np.stack([h - h0 for _, h in cols], axis=-1))
    K0 = torch.from_numpy(K0)
    idx, fs = _order(d6)
    inv = torch.from_numpy(np.argsort(idx))

    def solve(stage, term, G0, g0):
        p = torch.cat([t.reshape(B, -1) for t in (stage, term, G0, g0)], dim=-1)
        K = K0 + torch.einsum("ijp,bp->bij", dK, p)
        z = torch.linalg.solve(K, -torch.einsum("ip,bp->bi", dh, p))
        flat = z[:, inv]
        out, o = [], 0
        for k, n in zip(KEYS, fs):
            out.append(flat[:, o:o + n].reshape(aref._shapes(d6, B)[k]))
            o += n
        return tuple(out)
    return solve


def _setup(monkeypatch, case):
    torch = pytest.importorskip("torch")
    import aligator_b200.autograd as ag
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: types.SimpleNamespace(cuda_stream=0))
    s = _DenseHandle(torch, case)
    recs = [torch.from_numpy(np.ascontiguousarray(r)) for r in jacobian_records(case, 11)]
    solve = lambda *P: ag._Solve.apply(ag._Higher(s, MU), *P)
    ref = _torch_reference(torch, case, [r.numpy() for r in recs])
    g = torch.Generator().manual_seed(3)
    W = [torch.randn(o.shape, generator=g, dtype=torch.float64) for o in ref(*recs)]

    def loss(f):
        def L(*P):
            return sum((w * o).sum() + 0.5 * (w * o * o).sum() for w, o in zip(W, f(*P)))
        return L
    return torch, ag, s, recs, solve, ref, loss, g


def _close(torch, a, b, tol=1e-10):
    if isinstance(a, (tuple, list)):
        for x, y in zip(a, b):
            _close(torch, x, y, tol)
        return
    assert a.shape == b.shape, (a.shape, b.shape)
    scale = max(1.0, float(b.abs().max())) if b.numel() else 1.0
    assert float((a - b).abs().max()) <= tol * scale if a.numel() else True


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_values_grad_and_grad_of_grad(monkeypatch, case):
    torch, ag, s, recs, solve, ref, loss, g = _setup(monkeypatch, case)
    _close(torch, solve(*recs), ref(*recs))
    P = [r.clone().requires_grad_(True) for r in recs]
    Pr = [r.clone().requires_grad_(True) for r in recs]
    gs = torch.autograd.grad(loss(solve)(*P), P, create_graph=True)
    gr = torch.autograd.grad(loss(ref)(*Pr), Pr, create_graph=True)
    _close(torch, gs, gr)
    V = [torch.randn(r.shape, generator=g, dtype=torch.float64) for r in recs]
    hs = torch.autograd.grad(sum((a * v).sum() for a, v in zip(gs, V)), P)
    hr = torch.autograd.grad(sum((a * v).sum() for a, v in zip(gr, V)), Pr)
    _close(torch, hs, hr)


@pytest.mark.parametrize("case", CASES[:2], ids=IDS[:2])
def test_hessian_jvp_of_grad_and_third_order(monkeypatch, case):
    torch, ag, s, recs, solve, ref, loss, g = _setup(monkeypatch, case)
    F = torch.func
    for i in (0, 1):  # stage, term
        f = lambda x, f_=solve: loss(f_)(*[x if k == i else r for k, r in enumerate(recs)])
        fr = lambda x: loss(ref)(*[x if k == i else r for k, r in enumerate(recs)])
        s.calls.clear()
        H = F.hessian(f)(recs[i])
        counts = dict(s.calls)
        _close(torch, H, F.hessian(fr)(recs[i]))
        # one call per op and level, whatever the number of directions (recs[i] has dozens of entries): the sweep (its
        # backward, and no second one: the resolves find the factorisation current), the first-order pass (one
        # resolve, one gradient) and the HVP's (two rho, two resolves, one two-pair gradient)
        assert counts == HVP_CALLS, counts
        v = torch.randn(recs[i].shape, generator=g, dtype=torch.float64)
        V = torch.randn((3,) + tuple(recs[i].shape), generator=g, dtype=torch.float64)
        s.calls.clear()
        F.vmap(lambda d: F.jvp(F.grad(f), (recs[i],), (d,))[1])(V)
        assert s.calls == HVP_CALLS, s.calls
        _close(torch, F.jvp(F.grad(f), (recs[i],), (v,))[1], F.jvp(F.grad(fr), (recs[i],), (v,))[1])
        # a third derivative: the directional derivative of the Hessian-vector product (forward over forward over
        # reverse), against the reference's in reverse mode throughout
        w = torch.randn(recs[i].shape, generator=g, dtype=torch.float64)
        third = F.jvp(lambda x: F.jvp(F.grad(f), (x,), (w,))[1], (recs[i],), (v,))[1]
        want = F.grad(lambda x: (F.grad(lambda y: (F.grad(fr)(y) * w).sum())(x) * v).sum())(recs[i])
        _close(torch, third, want, 1e-9)
    # jacfwd(jacfwd) and jacrev(jacfwd) of one output with respect to term
    out = lambda f: (lambda t: f(recs[0], t, recs[2], recs[3])[0])
    want = F.jacrev(F.jacrev(out(ref)))(recs[1])
    _close(torch, F.jacfwd(F.jacfwd(out(solve)))(recs[1]), want)
    _close(torch, F.jacrev(F.jacfwd(out(solve)))(recs[1]), want)


def test_refusals(monkeypatch):
    torch, ag, s, recs, solve, ref, loss, g = _setup(monkeypatch, CASES[0])
    with pytest.raises(NotImplementedError, match="cotangents and tangents"):
        torch.func.vmap(lambda st: solve(st, *recs[1:]))(recs[0].expand(2, *recs[0].shape))
    with pytest.raises(NotImplementedError, match="cotangents and tangents"):  # the data of a resolve, vmapped
        _, vjp = torch.func.vjp(lambda st: solve(st, *recs[1:])[0], recs[0])
        torch.func.vmap(lambda st: ag._Resolve.apply(ag._Higher(s, MU), st, *recs[1:], recs[0].new_ones(
            s.shapes["xs"]), None, None, None, None, None))(recs[0].expand(2, *recs[0].shape))
    with pytest.raises(ValueError, match="CudaRiccatiBatch"):
        ag.lq_solve_higher(s, *recs, MU)
    import aligator_b200.gar as gar
    for kind in (dict(dense=True, nth=0, legs=0), dict(dense=False, nth=2, legs=0), dict(dense=False, nth=3, legs=2)):
        b = object.__new__(gar.CudaRiccatiBatch)
        b.__dict__.update(kind)
        with pytest.raises(ValueError, match="plain serial handles only"):
            ag.lq_solve_higher(b, *recs, MU)


@pytest.mark.parametrize("d6,B,mu", [((4, 2, 2, 0, 4, 6), 2, 1e-3), ((12, 6, 0, 0, 12, 3), 1, 1e-2)],
                         ids=["c3_mu1e-3", "c2"])
def test_hvp_references_agree(d6, B, mu):
    """The fp64 composition of the HVP on the oracle's solves (the e_ref of the GPU bar) against the independent
    extended-precision central differences of the gradient records (tests/hp_higher_order.py), on well-conditioned
    cases where the two must agree to a few hundred ulps (at small mu with terminal constraints the fp64 error grows
    like 1 / mu: that is what the GPU bar's e_ref measures)."""
    import hp_higher_order as hho
    import hp_reference as hp
    from lq_cases import symmetric_dot
    nx, nu, nc, nct, nc0, N = d6
    probs = gen.general_initial_condition(gen.generate_batch(3, B, N, nx, nu, nc, nct), nc0, 3)
    rng = np.random.default_rng(1)
    W = {k: rng.standard_normal(s) for k, s in aref._shapes(d6, B).items()}
    dot = symmetric_dot(rng, d6, B)
    e = hp.grad_errors(hho.hvp_fp64(hp.records(probs), d6, mu, W, dot), hho.hvp_hp(probs, mu, W, dot), d6)
    assert max(e.values()) <= 1e-11, e
