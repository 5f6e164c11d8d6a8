"""The tangent (forward mode) of the LQ solve on the GPU (ab2_gar_tangent, gar.h; the jvp of
aligator_b200.autograd.lq_solve): zdot against the oracle's solve of the numpy restatement's tangent problem
(lq_tangent_ref.py), the handle's state afterwards, exactness under zero / NULL / scaled tangents and repeated or
aliased calls, the per-instance-mu twin, cycle_append, the errors, the duality with the adjoint, torch.func.jvp,
gradcheck in forward mode and the full-size configurations."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import gen
import lq_adjoint_ref as aref
import lq_tangent_ref as ref
import test_gpu_adjoint as ga
from oracle import gar_oracle as orc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MU = 1e-2
MUS = (1.0, 1e-2, 1e-5)
TOL = 1e-10
KEYS = aref.KEYS
DOTS = ("stage", "term", "G0", "g0")
HANDLES = ga.HANDLES
FEW = [HANDLES[0], HANDLES[9], HANDLES[-3], HANDLES[-2], HANDLES[-1]]
FEW_IDS = ["lane_v0", "mma_12_v7", "cta_v9", "cta_runtime", "dense"]


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import __graft_entry__ as g
    g.build()
    import aligator_b200.gar as gar
    import aligator_b200.autograd as ag
    return gar, ag, torch


def _tangent(env, s, seed, scale=1.0):
    """A random data tangent in the problem's layouts (asymmetric Q, R blocks, nonzero pad double)."""
    _, _, torch = env
    d = s.dims
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    shapes = dict(stage=(d.batch, d.horizon, s.srec), term=(d.batch, s.trec), G0=(d.batch, d.nc0 * d.nx),
                  g0=(d.batch, d.nc0))
    return {k: scale * torch.randn(v, generator=g, dtype=torch.float64, device="cuda") for k, v in shapes.items()}


def _np(d):
    return {k: None if v is None else v.cpu().numpy() for k, v in d.items()}


def _zdot(env, s):
    return _np(ga._primal(env, s))


def _oracle_solve(recs, dims, mu):
    nx, nu, nc, nct, nc0, N, B = dims
    bo = orc.BatchedOracle(nx, nu, nc, nct, nc0, N, B, *[np.ascontiguousarray(a) for a in recs])
    bo.sweep(mu, nthreads=1)
    assert np.all(bo.status == 1)  # the oracle reports 1 = ok
    return aref.oracle_dict(bo.get())


def _oracle_tangent(recs, dot, dims, mu):
    d6 = dims[:6]
    z = _oracle_solve(recs, dims, mu)
    return _oracle_solve(ref.tangent_records(*recs, dot, z, d6), dims, mu)


def _check_against_oracle(got, want, tag):
    for k in KEYS:
        if np.asarray(want[k]).size:
            e = gen.rel_fro(got[k], want[k])
            assert e <= TOL, (tag, k, e)


def _equal(a, b):
    return all(np.array_equal(a[k], b[k]) for k in KEYS)


@pytest.mark.parametrize("mu", MUS, ids=["mu1", "mu1e-2", "mu1e-5"])
@pytest.mark.parametrize("name,kw,dims", HANDLES, ids=[h[0] for h in HANDLES])
def test_tangent_matches_oracle_and_state_afterwards(env, name, kw, dims, mu):
    gar, _, torch = env
    s, recs = ga._setup(env, kw, dims, seed=dims[0] * 31 + dims[-1], mu=mu)
    before = ga._outputs(gar, s)
    problem = [s.get_problem(w).copy() for w in range(4)]
    primal = ga._primal(env, s)
    dot = _tangent(env, s, 1)
    n0 = s.launch_count()
    s.tangent(primal, dot, mu)
    s.synchronize()
    assert s.launch_count() - n0 == 3
    _check_against_oracle(_zdot(env, s), _oracle_tangent(recs, _np(dot), dims, mu), (name, mu))
    # the matrix recursion never reads the vectors: FB, VXX and the pivot statistics are the primal sweep's
    after = ga._outputs(gar, s)
    for k in (gar.OUT_FB, gar.OUT_VXX, gar.OUT_FBT, "pivots", "status"):
        if k in before:
            assert np.array_equal(after[k], before[k]), (name, k)
    for w in range(4):
        assert np.array_equal(s.get_problem(w), problem[w]), (name, "problem", w)
    s.sweep(mu)
    again = ga._outputs(gar, s)
    for k in before:
        assert np.array_equal(again[k], before[k], equal_nan=True), (name, "sweep after tangent", k)
    s.close()


@pytest.mark.parametrize("name,kw,dims", FEW, ids=FEW_IDS)
def test_exactness(env, name, kw, dims):
    gar, _, torch = env
    s, _ = ga._setup(env, kw, dims, seed=5)
    primal = ga._primal(env, s)
    dot = _tangent(env, s, 2)
    s.tangent(primal, dot, MU)
    base = _zdot(env, s)
    # two identical calls: identical bits
    s.tangent(primal, dot, MU)
    assert _equal(_zdot(env, s), base), name
    # a zero tangent and an all-NULL tangent: exact zeros
    for zero in ({k: torch.zeros_like(v) for k, v in dot.items()}, {}, {k: None for k in DOTS}):
        s.tangent(primal, zero, MU)
        for k, v in _zdot(env, s).items():
            assert np.all(v == 0.0), (name, "zero", k)
    # a tangent scaled by 2^k: exactly 2^k zdot
    for e in (-40, 7, 40):
        s.tangent(primal, {k: v * 2.0 ** e for k, v in dot.items()}, MU)
        got = _zdot(env, s)
        for k in KEYS:
            assert np.array_equal(got[k], base[k] * 2.0 ** e), (name, e, k)
    # NULL tangent fields: the same bits as explicit zero arrays
    for drop in (("stage",), ("term", "g0"), ("G0",)):
        s.tangent(primal, {k: (None if k in drop else v) for k, v in dot.items()}, MU)
        a = _zdot(env, s)
        s.tangent(primal, {k: (torch.zeros_like(v) if k in drop else v) for k, v in dot.items()}, MU)
        assert _equal(a, _zdot(env, s)), (name, drop)
    # the primal passed as the handle's own outputs: the same bits as a copy
    s.sweep(MU)
    own = {k: s.device_ptr(w) for k, w in ga._out_of(gar).items()}
    s.tangent(own, dot, MU)
    assert _equal(_zdot(env, s), base), (name, "aliased primal")
    s.close()


@pytest.mark.parametrize("name,kw,dims", FEW, ids=FEW_IDS)
def test_tangent_v_matches_scalar_calls(env, name, kw, dims):
    gar, _, torch = env
    nx, nu, nc, nct, nc0, N, B = dims
    s, _ = ga._setup(env, kw, dims, seed=9)
    dot = _tangent(env, s, 3)
    # a constant array: the scalar call's bits
    primal = ga._primal(env, s)
    s.tangent(primal, dot, MU)
    want = _zdot(env, s)
    for mu_arg in (np.full(B, MU), torch.full((B,), MU, dtype=torch.float64, device="cuda")):
        n0 = s.launch_count()
        s.tangent(primal, dot, mu_arg)
        s.synchronize()
        assert s.launch_count() - n0 == 3
        assert _equal(_zdot(env, s), want), (name, "constant", type(mu_arg))
    # distinct mu_b: instance b as in the scalar call at mu_b
    mu_b = np.array([MUS[b % 3] for b in range(B)])
    want = {k: np.empty(v.shape) for k, v in want.items()}
    want_out = {}
    for v in MUS:
        s.sweep(v)
        s.tangent(ga._primal(env, s), dot, v)
        sel = mu_b == v
        for k, a in _zdot(env, s).items():
            want[k][sel] = a[sel]
        for k, a in ga._outputs(gar, s).items():
            want_out.setdefault(k, np.empty_like(a))[sel] = a[sel]
    for mu_arg in (mu_b, torch.tensor(mu_b, device="cuda")):
        s.sweep(mu_arg)
        s.tangent(ga._primal(env, s), dot, mu_arg)
        assert _equal(_zdot(env, s), want), (name, type(mu_arg))
        got_out = ga._outputs(gar, s)
        for k in want_out:
            assert np.array_equal(got_out[k], want_out[k], equal_nan=True), (name, type(mu_arg), k)
    s.close()


# (not the dense handle: its sweep kernel reads the solver-owned stage records without the ring head, DESIGN §8)
@pytest.mark.parametrize("name,kw,dims", FEW[:4], ids=FEW_IDS[:4])
def test_cycle_append_then_tangent(env, name, kw, dims):
    gar, _, torch = env
    nx, nu, nc, nct, nc0, N, B = dims
    s, recs = ga._setup(env, kw, dims, seed=13)
    new_last = np.ascontiguousarray(gar.pack_problems(gen.generate_batch(99, B, 1, nx, nu, nc, nct))[0].reshape(B, -1))
    s.cycle_append(new_last)
    s.sweep(MU)
    primal = ga._primal(env, s)
    dot = _tangent(env, s, 4)
    s.tangent(primal, dot, MU)
    got, got_out = _zdot(env, s), ga._outputs(gar, s)
    rot = np.ascontiguousarray(np.concatenate([recs[0].reshape(B, N, -1)[:, 1:], new_last[:, None]], axis=1))
    f = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
    f.set_problem(rot, recs[1], recs[2], recs[3])
    f.sweep(MU)
    f.tangent(ga._primal(env, f), dot, MU)
    assert _equal(got, _zdot(env, f)), name
    for k, a in ga._outputs(gar, f).items():
        assert np.array_equal(got_out[k], a, equal_nan=True), (name, k)
    s.close()
    f.close()


def _rc(gar, s, primal, dot, mu=MU):
    pr = gar._fill(gar.LsIterate(), gar._LS_KEYS, primal)
    dt = gar._fill(gar.LqTangent(), gar._GRAD_KEYS, dot)
    return gar.lib().ab2_gar_tangent(s.h, C.c_double(mu), C.byref(pr), C.byref(dt), None)


def test_errors(env):
    gar, _, torch = env
    nx, nu, nc, nct, nc0, N, B = 5, 2, 1, 1, 5, 5, 7
    for kw in (dict(nth=2), dict(legs=3)):
        s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
        stage, term, G0, g0 = gar.pack_problems(gen.generate_batch(1, B, N, nx, nu, nc, nct))
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
        z = ga._zeros_like_outputs(env, s)
        assert _rc(gar, s, z, {}) == 2, kw  # AB2_ERR_UNSUPPORTED
        with pytest.raises(gar.GarError):
            s.tangent(z, {}, MU)
        assert s.launch_count() == n0
        s.close()
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    z = ga._zeros_like_outputs(env, s)
    assert _rc(gar, s, z, {}) == 4  # AB2_ERR_STATE: no problem set
    assert s.launch_count() == 0
    s.set_problem(*gar.pack_problems(gen.generate_batch(1, B, N, nx, nu, nc, nct)))
    s.sweep(MU)
    s.synchronize()
    n0 = s.launch_count()
    for k in KEYS:
        missing = dict(z)
        missing[k] = None
        assert _rc(gar, s, missing, {}) == 1, k  # AB2_ERR_INVALID
    assert _rc(gar, s, z, {}, mu=0.0) == 1  # constraints need mu > 0
    assert s.launch_count() == n0
    s.close()


@pytest.mark.parametrize("name,kw,dims", FEW[:3], ids=FEW_IDS[:3])
def test_duality_with_the_adjoint(env, name, kw, dims):
    """<zbar, tangent(pdot)> = <adjoint(zbar), pdot> on the device."""
    gar, _, torch = env
    s, _ = ga._setup(env, kw, dims, seed=17)
    primal = ga._primal(env, s)
    zbar = ga._cotangent(env, s, 6)
    dot = _tangent(env, s, 7)
    grad = ga._grad_bufs(env, s)
    s.adjoint(primal, zbar, grad, MU)
    s.tangent(primal, dot, MU)
    zdot = ga._primal(env, s)
    lhs = sum(float(torch.sum(zbar[k] * zdot[k])) for k in KEYS)
    rhs = sum(float(torch.sum(grad[k] * dot[k])) for k in DOTS)
    assert abs(lhs - rhs) <= 1e-12 * max(abs(lhs), abs(rhs)), (name, lhs, rhs)
    s.close()


def test_func_jvp_is_the_tangent_call(env):
    gar, ag, torch = env
    name, kw, dims = HANDLES[0]
    nx, nu, nc, nct, nc0, N, B = dims
    s, recs = ga._setup(env, kw, dims, seed=23)
    prim = tuple(torch.tensor(np.ascontiguousarray(a), device="cuda") for a in recs)
    dot = _tangent(env, s, 8)
    tans = tuple(dot[k] for k in DOTS)
    outs, jv = torch.func.jvp(lambda *a: ag.lq_solve(s, *a, MU), prim, tans)
    s.set_problem(*prim, memspace=gar.AB2_DEVICE)
    s.sweep(MU)
    primal = ga._primal(env, s)
    for k, o in zip(KEYS, outs):
        assert torch.equal(o, primal[k]), k
    s.tangent(primal, dot, MU)
    want = ga._primal(env, s)
    for k, t in zip(KEYS, jv):
        assert torch.equal(t, want[k]), k
    # torch.autograd.forward_ad gives the same bits
    import torch.autograd.forward_ad as fwAD
    with fwAD.dual_level():
        o = ag.lq_solve(s, *[fwAD.make_dual(p, t) for p, t in zip(prim, tans)], MU)
        for k, y in zip(KEYS, o):
            assert torch.equal(fwAD.unpack_dual(y).tangent, want[k]), k
    s.close()


@pytest.mark.parametrize("dims,kw", [((4, 2, 2, 1, 4, 3, 2), {}), ((7, 3, 2, 1, 7, 2, 2), {})],
                         ids=["warp", "cta_runtime"])
def test_gradcheck_forward_mode(env, dims, kw):
    gar, ag, torch = env
    nx, nu, nc, nct, nc0, N, B = dims
    probs = gen.generate_batch(21, B, N, nx, nu, nc, nct)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
    blocks, term, init = ga._block_inputs(torch, probs)
    names = list(blocks) + ["t" + n for n in term] + list(init)
    leaves = list(blocks.values()) + list(term.values()) + list(init.values())
    sym = lambda P: 0.5 * (P + P.transpose(-1, -2))

    def f(*xs):
        a = dict(zip(names, xs))
        st = ag.stage_records(a["A"], a["B"], a["f"], sym(a["Q"]), a["S"], sym(a["R"]), a["q"], a["r"], a["C"], a["D"],
                              a["d"])
        tt = ag.term_records(sym(a["tQ"]), a["tq"], a["tC"], a["td"])
        return ag.lq_solve(s, st.contiguous(), tt.contiguous(), a["G0"], a["g0"], MU)

    assert torch.autograd.gradcheck(f, tuple(leaves), eps=1e-6, atol=1e-6, rtol=1e-4, check_forward_ad=True,
                                    check_backward_ad=False)
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
    primal = ga._primal(env, s)
    dot = _tangent(env, s, 5)
    s.tangent(primal, dot, mu)
    s.synchronize()
    assert np.all(s.status() == 0)
    got = _zdot(env, s)
    idx = np.r_[0:4, B // 2 - 2:B // 2 + 2, B - 8:B]  # first wave, a wave boundary, the ragged tail
    sub = lambda t: np.ascontiguousarray(t.cpu().numpy()[idx])
    recs = [sub(t) for t in (stage, term, G0, g0)]
    dims = (nx, nu, nc, nct, nx, N, len(idx))
    want = _oracle_tangent(recs, {k: sub(v) for k, v in dot.items()}, dims, mu)
    _check_against_oracle({k: v[idx] for k, v in got.items()}, want, name)
    s.close()
