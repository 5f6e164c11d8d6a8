"""The adjoint of the LQ solve on the GPU (ab2_gar_adjoint, gar.h; aligator_b200.autograd.lq_solve): gradients against
the numpy restatement (lq_adjoint_ref.py) applied to the oracle's primal and adjoint solves, the handle's state
afterwards, exactness under zero / scaled / NULL cotangents, the per-instance-mu twin, cycle_append, the errors,
torch.autograd.gradcheck and the full-size configurations."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import gen
import lq_adjoint_ref as ref
from oracle import gar_oracle as orc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MU = 1e-2
MUS = (1.0, 1e-2, 1e-5)
TOL = 1e-10
OUTS_PLAIN = range(13)  # OUT_FF .. OUT_LBDAS
KEYS = ref.KEYS
GRADS = ("stage", "term", "G0", "g0")


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import __graft_entry__ as g
    g.build()
    import aligator_b200.gar as gar
    import aligator_b200.autograd as ag
    return gar, ag, torch


# (name, CudaRiccatiBatch keyword arguments, (nx, nu, nc, nct, nc0, N, B))
HANDLES = [("lane_v%d" % v, dict(variant=v), (4, 2, 2, 2, 4, 6, 9)) for v in range(7)] + [
    ("lane_12_6_6", {}, (12, 6, 6, 3, 12, 5, 7))] + [
    ("mma_12_v%d" % v, dict(variant=v), (12, 6, 0, 3, 12, 6, 9)) for v in (6, 7, 8, 10)] + [
    ("mma_14_v%d" % v, dict(variant=v), (14, 7, 0, 2, 14, 4, 5)) for v in (6, 7, 8, 10)] + [
    ("cta_v9", dict(variant=9), (4, 2, 2, 2, 4, 6, 9)),
    ("cta_runtime", {}, (7, 3, 2, 2, 7, 5, 8)),
    ("dense", dict(dense=True), (4, 2, 2, 2, 4, 5, 8)),
]


def _dev(torch, a):
    return torch.tensor(np.ascontiguousarray(a, dtype=np.float64), device="cuda")


def _empty(torch, s, w):
    return torch.empty(s.out_shape(w), dtype=torch.float64, device="cuda")


def _out_of(gar):
    return dict(xs=gar.OUT_XS, us=gar.OUT_US, vs=gar.OUT_VS, vsT=gar.OUT_VST, lam0=gar.OUT_LBD0, lams=gar.OUT_LBDAS)


def _primal(env, s):
    """The handle's trajectory copied into tensors of the caller (what the last sweep returned)."""
    gar, _, torch = env
    out = {}
    for k, w in _out_of(gar).items():
        t = _empty(torch, s, w)
        if t.numel():
            s.get_into(w, t, gar.AB2_DEVICE)
        out[k] = t
    s.synchronize()
    return out


def _cotangent(env, s, seed, scale=1.0):
    gar, _, torch = env
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return {k: scale * torch.randn(s.out_shape(w), generator=g, dtype=torch.float64, device="cuda")
            for k, w in _out_of(gar).items()}


def _grad_bufs(env, s, fill=float("nan")):
    _, _, torch = env
    d = s.dims
    shapes = dict(stage=(d.batch, d.horizon, s.srec), term=(d.batch, s.trec), G0=(d.batch, d.nc0 * d.nx),
                  g0=(d.batch, d.nc0))
    return {k: torch.full(v, fill, dtype=torch.float64, device="cuda") for k, v in shapes.items()}


def _np(d):
    return {k: v.cpu().numpy() for k, v in d.items()}


def _outputs(gar, s):
    r = {w: s.get(w).copy() for w in OUTS_PLAIN if int(np.prod(s.out_shape(w)))}
    r["status"] = s.status().copy()
    r["pivots"] = np.stack(s.pivot_stats(), axis=1)
    return r


def _setup(env, kw, dims, seed, mu=MU):
    gar, _, _ = env
    nx, nu, nc, nct, nc0, N, B = dims
    probs = gen.generate_batch(seed, B, N, nx, nu, nc, nct)
    recs = [np.ascontiguousarray(a) for a in gar.pack_problems(probs)]
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
    s.set_problem(*recs)
    s.sweep(mu)
    return s, recs


def _oracle_grads(recs, cot, dims, mu):
    """Numpy gradients from the oracle's primal solve and its solve of the adjoint problem."""
    nx, nu, nc, nct, nc0, N, B = dims
    d6 = (nx, nu, nc, nct, nc0, N)

    def solve(st, tt, G0, g0):
        bo = orc.BatchedOracle(nx, nu, nc, nct, nc0, N, B, st, tt, G0, g0)
        bo.sweep(mu, nthreads=1)
        assert np.all(bo.status == 1)  # the oracle reports 1 = ok
        return ref.oracle_dict(bo.get())

    z = solve(*recs)
    w = solve(*ref.adjoint_records(*recs, cot, d6))
    return ref.grad_records(z, w, d6)


def _families(g, dims):
    """Gradient records -> {family: array over instances and knots}."""
    nx, nu, nc, nct, nc0, N, B = dims
    so, _ = ref.stage_offsets(nx, nu, nc)
    to, _ = ref.term_offsets(nx, nct)
    st = np.asarray(g["stage"]).reshape(B, N, -1)
    tt = np.asarray(g["term"]).reshape(B, -1)
    fam = {n: st[..., a:b] for n, (a, b) in so.items()}
    fam.update({"term_" + n: tt[:, a:b] for n, (a, b) in to.items()})
    fam["G0"], fam["g0"] = np.asarray(g["G0"]).reshape(B, -1), np.asarray(g["g0"]).reshape(B, -1)
    fam["pad"] = st[..., sum(b - a for a, b in so.values()):]
    return fam


def _check_against_oracle(got, want, dims, tag):
    gf, wf = _families(got, dims), _families(want, dims)
    for n in wf:
        if n == "pad":
            assert np.all(gf[n] == 0.0), (tag, "pad")
        elif wf[n].size:
            e = gen.rel_fro(gf[n], wf[n])
            assert e <= TOL, (tag, n, e)


@pytest.mark.parametrize("name,kw,dims", HANDLES, ids=[h[0] for h in HANDLES])
def test_gradients_match_oracle_and_state_afterwards(env, name, kw, dims):
    gar, _, torch = env
    s, recs = _setup(env, kw, dims, seed=dims[0] * 31 + dims[-1])
    before = _outputs(gar, s)
    problem = [s.get_problem(w).copy() for w in range(4)]
    primal = _primal(env, s)
    cot = _cotangent(env, s, 1)
    grad = _grad_bufs(env, s)
    n0 = s.launch_count()
    s.adjoint(primal, cot, grad, MU)
    s.synchronize()
    assert s.launch_count() - n0 == 3
    got = _np(grad)
    _check_against_oracle(got, _oracle_grads(recs, _np(cot), dims, MU), dims, name)
    # the matrix recursion never reads the vectors: FB, VXX and the pivot statistics are the primal sweep's
    after = _outputs(gar, s)
    for k in (gar.OUT_FB, gar.OUT_VXX, gar.OUT_FBT, "pivots", "status"):
        if k in before:
            assert np.array_equal(after[k], before[k]), (name, k)
    # ... while the trajectory is the adjoint solution w
    assert not np.array_equal(after[gar.OUT_XS], before[gar.OUT_XS])
    for w in range(4):
        assert np.array_equal(s.get_problem(w), problem[w]), (name, "problem", w)
    s.sweep(MU)
    again = _outputs(gar, s)
    for k in before:
        assert np.array_equal(again[k], before[k], equal_nan=True), (name, "sweep after adjoint", k)
    s.close()


@pytest.mark.parametrize("name,kw,dims", [HANDLES[0], HANDLES[9], HANDLES[-3], HANDLES[-2], HANDLES[-1]],
                         ids=["lane_v0", "mma_12_v7", "cta_v9", "cta_runtime", "dense"])
def test_exactness(env, name, kw, dims):
    gar, _, torch = env
    s, _ = _setup(env, kw, dims, seed=5)
    primal = _primal(env, s)
    cot = _cotangent(env, s, 2)
    base = _grad_bufs(env, s)
    s.adjoint(primal, cot, base, MU)
    base = _np(base)
    # zero cotangents: all-zero gradients
    zero = _grad_bufs(env, s)
    s.adjoint(primal, {k: torch.zeros_like(v) for k, v in cot.items()}, zero, MU)
    for k, v in _np(zero).items():
        assert np.all(v == 0.0), (name, "zero", k)
    # cotangents scaled by 2^k: gradients exactly 2^k times as large
    for e in (-40, 7, 40):
        g = _grad_bufs(env, s)
        s.adjoint(primal, {k: v * 2.0 ** e for k, v in cot.items()}, g, MU)
        for k, v in _np(g).items():
            assert np.array_equal(v, base[k] * 2.0 ** e), (name, e, k)
    # NULL cotangent fields: the same bits as explicit zero arrays
    for drop in (("vs", "lam0"), ("xs",), ("us", "vsT", "lams")):
        part = {k: (None if k in drop else v) for k, v in cot.items()}
        expl = {k: (torch.zeros_like(v) if k in drop else v) for k, v in cot.items()}
        a, b = _grad_bufs(env, s), _grad_bufs(env, s)
        s.adjoint(primal, part, a, MU)
        s.adjoint(primal, expl, b, MU)
        for k in GRADS:
            assert np.array_equal(_np(a)[k], _np(b)[k]), (name, drop, k)
    # NULL gradient outputs are not written; the requested ones are as in the full call
    for want in (("stage",), ("term", "g0"), ("G0",)):
        bufs = _grad_bufs(env, s)
        big = torch.full((bufs["stage"].numel() + 64,), float("nan"), dtype=torch.float64, device="cuda")
        bufs["stage"] = big[32:32 + bufs["stage"].numel()].view(bufs["stage"].shape)
        s.adjoint(primal, cot, {k: bufs[k] for k in want}, MU)
        s.synchronize()
        for k in GRADS:
            v = bufs[k].cpu().numpy()
            if k in want:
                assert np.array_equal(v, base[k]), (name, want, k)
            elif v.size:
                assert np.all(np.isnan(v)), (name, want, k)
        guard = big.cpu().numpy()
        assert np.all(np.isnan(guard[:32])) and np.all(np.isnan(guard[-32:])), (name, want)
    s.close()


@pytest.mark.parametrize("name,kw,dims", [HANDLES[0], HANDLES[9], HANDLES[-3], HANDLES[-2], HANDLES[-1]],
                         ids=["lane_v0", "mma_12_v7", "cta_v9", "cta_runtime", "dense"])
def test_adjoint_v_matches_scalar_calls(env, name, kw, dims):
    gar, _, torch = env
    nx, nu, nc, nct, nc0, N, B = dims
    s, _ = _setup(env, kw, dims, seed=9)
    mu_b = np.array([MUS[b % 3] for b in range(B)])
    cot = _cotangent(env, s, 3)
    want = {k: np.empty(v.shape) for k, v in _grad_bufs(env, s).items()}
    want_out = {}
    for v in MUS:
        s.sweep(v)
        primal = _primal(env, s)
        g = _grad_bufs(env, s)
        s.adjoint(primal, cot, g, v)
        sel = mu_b == v
        for k, a in _np(g).items():
            want[k][sel] = a[sel]
        for k, a in _outputs(gar, s).items():
            want_out.setdefault(k, np.empty_like(a))[sel] = a[sel]
    for mu_arg in (mu_b, torch.tensor(mu_b, device="cuda")):
        s.sweep(mu_arg)
        primal = _primal(env, s)
        g = _grad_bufs(env, s)
        n0 = s.launch_count()
        s.adjoint(primal, cot, g, mu_arg)
        s.synchronize()
        assert s.launch_count() - n0 == 3
        for k, a in _np(g).items():
            assert np.array_equal(a, want[k]), (name, type(mu_arg), k)
        got_out = _outputs(gar, s)
        for k in want_out:
            assert np.array_equal(got_out[k], want_out[k], equal_nan=True), (name, type(mu_arg), k)
    s.close()


# (not the dense handle: its sweep kernel reads the solver-owned stage records in physical order, without the ring
# head cycle_append advances, so its primal sweep after cycle_append is not the rotated problem's)
@pytest.mark.parametrize("name,kw,dims", [HANDLES[0], HANDLES[9], HANDLES[-3], HANDLES[-2]],
                         ids=["lane_v0", "mma_12_v7", "cta_v9", "cta_runtime"])
def test_cycle_append_then_adjoint(env, name, kw, dims):
    gar, _, torch = env
    nx, nu, nc, nct, nc0, N, B = dims
    s, recs = _setup(env, kw, dims, seed=13)
    new_last = np.ascontiguousarray(gar.pack_problems(gen.generate_batch(99, B, 1, nx, nu, nc, nct))[0].reshape(B, -1))
    s.cycle_append(new_last)
    s.sweep(MU)
    primal = _primal(env, s)
    cot = _cotangent(env, s, 4)
    g = _grad_bufs(env, s)
    s.adjoint(primal, cot, g, MU)
    got, got_out = _np(g), _outputs(gar, s)
    rot = np.ascontiguousarray(np.concatenate([recs[0].reshape(B, N, -1)[:, 1:], new_last[:, None]], axis=1))
    f = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
    f.set_problem(rot, recs[1], recs[2], recs[3])
    f.sweep(MU)
    primal_f = _primal(env, f)
    for k in KEYS:
        assert torch.equal(primal_f[k], primal[k]), (name, k)
    gf = _grad_bufs(env, f)
    f.adjoint(primal_f, cot, gf, MU)
    for k, a in _np(gf).items():
        assert np.array_equal(got[k], a), (name, k)
    for k, a in _outputs(gar, f).items():
        assert np.array_equal(got_out[k], a, equal_nan=True), (name, k)
    s.close()
    f.close()


def _rc(gar, s, primal, cot, grad, mu=MU):
    pr = gar._fill(gar.LsIterate(), gar._LS_KEYS, primal)
    ct = gar._fill(gar.LsIterate(), gar._LS_KEYS, cot)
    gr = gar._fill(gar.LqGrad(), gar._GRAD_KEYS, grad)
    return gar.lib().ab2_gar_adjoint(s.h, C.c_double(mu), C.byref(pr), C.byref(ct), C.byref(gr), None)


def _zeros_like_outputs(env, s):
    gar, _, torch = env
    return {k: torch.zeros(s.out_shape(w), dtype=torch.float64, device="cuda") for k, w in _out_of(gar).items()}


def test_errors(env):
    gar, _, torch = env
    nx, nu, nc, nct, nc0, N, B = 5, 2, 1, 1, 5, 5, 7
    for kw in (dict(nth=2), dict(legs=3)):
        s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
        probs = gen.generate_batch(1, B, N, nx, nu, nc, nct)
        stage, term, G0, g0 = gar.pack_problems(probs)
        if s.nth and not s.legs:  # parametric records: the plain ones with zero parameter blocks
            st = np.zeros((B, N, s.srec))
            st[..., :stage.shape[-1]] = stage.reshape(B, N, -1)
            tt = np.zeros((B, s.trec))
            tt[:, :term.shape[1]] = term
            stage, term = st, tt
        s.set_problem(stage, term, G0, g0)
        s.sweep(MU)
        s.synchronize()
        n0 = s.launch_count()
        z = _zeros_like_outputs(env, s)
        assert _rc(gar, s, z, z, _grad_bufs(env, s)) == 2, kw  # AB2_ERR_UNSUPPORTED
        with pytest.raises(gar.GarError):
            s.adjoint(z, z, _grad_bufs(env, s), MU)
        assert s.launch_count() == n0
        s.close()
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    z = _zeros_like_outputs(env, s)
    assert _rc(gar, s, z, z, _grad_bufs(env, s)) == 4  # AB2_ERR_STATE: no problem set
    assert s.launch_count() == 0
    probs = gen.generate_batch(1, B, N, nx, nu, nc, nct)
    s.set_problem(*gar.pack_problems(probs))
    s.sweep(MU)
    s.synchronize()
    n0 = s.launch_count()
    alias = dict(z)
    alias["xs"] = s.device_ptr(gar.OUT_XS)  # the primal would be overwritten by the adjoint sweep
    assert _rc(gar, s, alias, z, _grad_bufs(env, s)) == 1
    inner = dict(z)
    inner["lams"] = s.device_ptr(gar.OUT_LBDAS) + 8 * nx  # overlapping, not at the start
    assert _rc(gar, s, inner, z, _grad_bufs(env, s)) == 1
    missing = dict(z)
    missing["us"] = None
    assert _rc(gar, s, missing, z, _grad_bufs(env, s)) == 1
    assert _rc(gar, s, z, z, _grad_bufs(env, s), mu=0.0) == 1  # constraints need mu > 0
    assert s.launch_count() == n0
    s.close()


def _block_inputs(torch, probs):
    """Leaf tensors of every block of a batch, Q and R as P with Q = (P + P^T) / 2."""
    N = probs[0].horizon
    T = lambda f: torch.tensor(np.stack([np.stack([np.asarray(f(p, t)) for t in range(N)]) for p in probs]),
                               dtype=torch.float64, device="cuda", requires_grad=True)
    blocks = {n: T(lambda p, t, n=n: getattr(p.stages[t], n)) for n in ("A", "B", "f", "Q", "S", "R", "q", "r", "C",
                                                                      "D", "d")}
    Tt = lambda f: torch.tensor(np.stack([np.asarray(f(p)) for p in probs]), dtype=torch.float64, device="cuda",
                                requires_grad=True)
    term = {n: Tt(lambda p, n=n: getattr(p.stages[N], n)) for n in ("Q", "q", "C", "d")}
    init = dict(G0=Tt(lambda p: np.asarray(p.G0).ravel(order="F")), g0=Tt(lambda p: p.g0))
    return blocks, term, init


@pytest.mark.parametrize("dims,kw", [((4, 2, 2, 1, 4, 3, 2), {}), ((7, 3, 2, 1, 7, 2, 2), {})],
                         ids=["warp", "cta_runtime"])
def test_gradcheck_lq_solve(env, dims, kw):
    gar, ag, torch = env
    nx, nu, nc, nct, nc0, N, B = dims
    probs = gen.generate_batch(21, B, N, nx, nu, nc, nct)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
    blocks, term, init = _block_inputs(torch, probs)
    names = list(blocks) + ["t" + n for n in term] + list(init)
    leaves = list(blocks.values()) + list(term.values()) + list(init.values())
    sym = lambda P: 0.5 * (P + P.transpose(-1, -2))

    def f(*xs):
        a = dict(zip(names, xs))
        st = ag.stage_records(a["A"], a["B"], a["f"], sym(a["Q"]), a["S"], sym(a["R"]), a["q"], a["r"], a["C"], a["D"],
                              a["d"])
        tt = ag.term_records(sym(a["tQ"]), a["tq"], a["tC"], a["td"])
        return ag.lq_solve(s, st.contiguous(), tt.contiguous(), a["G0"], a["g0"], MU)

    outs = f(*leaves)
    z = {k: o.detach().cpu().numpy() for k, o in zip(KEYS, outs)}
    dense = ref.solution_dict([gen.lqr_dense_solve(p, MU) for p in probs], (nx, nu, nc, nct, nc0, N))
    for k in KEYS:
        if dense[k].size:
            assert gen.rel_fro(z[k], dense[k]) <= 1e-9, k
    assert torch.autograd.gradcheck(f, tuple(leaves), eps=1e-6, atol=1e-6, rtol=1e-4)
    s.close()


@pytest.mark.parametrize("cfg", [("C2", 12, 6, 0, 0, 100, 4096, 1e-2), ("C3", 4, 2, 2, 0, 100, 16384, 1e-3)],
                         ids=["C2", "C3"])
def test_full_size(env, cfg):
    gar, _, torch = env
    sys.path.insert(0, ROOT)
    import bench
    name, nx, nu, nc, nct, N, B, mu = cfg
    stage, term, G0, g0 = bench.synth_batch_torch(torch, B, N, nx, nu, "cuda:0", 77, nc, nct, "control")
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nx, N, B)
    s.set_problem(stage, term, G0, g0, memspace=gar.AB2_DEVICE)
    s.sweep(mu)
    primal = _primal(env, s)
    cot = _cotangent(env, s, 5)
    grad = _grad_bufs(env, s)
    s.adjoint(primal, cot, grad, mu)
    s.synchronize()
    assert np.all(s.status() == 0)
    idx = np.r_[0:4, B // 2 - 2:B // 2 + 2, B - 8:B]  # first wave, a wave boundary, the ragged tail
    sub = lambda t: np.ascontiguousarray(t.cpu().numpy()[idx])
    recs = [sub(t) for t in (stage, term, G0, g0)]
    dims = (nx, nu, nc, nct, nx, N, len(idx))
    want = _oracle_grads(recs, {k: v.cpu().numpy()[idx] for k, v in cot.items()}, dims, mu)
    _check_against_oracle({k: sub(v) for k, v in grad.items()}, want, dims, name)
    s.close()
