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
import lq_gpu
from lq_gpu import HANDLES, MUS
from oracle import gar_oracle as orc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MU = 1e-2
TOL = 1e-10
KEYS = ref.KEYS
GRADS = ("stage", "term", "G0", "g0")


@pytest.fixture(scope="module")
def env():
    return lq_gpu.gpu_env()


def _dev(torch, a):
    return torch.tensor(np.ascontiguousarray(a, dtype=np.float64), device="cuda")


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
    s, recs = lq_gpu.setup(env, kw, dims, seed=dims[0] * 31 + dims[-1])
    before = lq_gpu.outputs(gar, s)
    problem = [s.get_problem(w).copy() for w in range(4)]
    primal = lq_gpu.primal(env, s)
    cot = lq_gpu.cotangent(env, s, 1)
    grad = lq_gpu.grad_bufs(env, s)
    n0 = s.launch_count()
    s.adjoint(primal, cot, grad, MU)
    s.synchronize()
    assert s.launch_count() - n0 == 3
    got = lq_gpu.to_np(grad)
    _check_against_oracle(got, _oracle_grads(recs, lq_gpu.to_np(cot), dims, MU), dims, name)
    # the matrix recursion never reads the vectors: FB, VXX and the pivot statistics are the primal sweep's
    after = lq_gpu.outputs(gar, s)
    for k in (gar.OUT_FB, gar.OUT_VXX, gar.OUT_FBT, "pivots", "status"):
        if k in before:
            assert np.array_equal(after[k], before[k]), (name, k)
    # ... while the trajectory is the adjoint solution w
    assert not np.array_equal(after[gar.OUT_XS], before[gar.OUT_XS])
    for w in range(4):
        assert np.array_equal(s.get_problem(w), problem[w]), (name, "problem", w)
    s.sweep(MU)
    again = lq_gpu.outputs(gar, s)
    for k in before:
        assert np.array_equal(again[k], before[k], equal_nan=True), (name, "sweep after adjoint", k)
    s.close()


@pytest.mark.parametrize("name,kw,dims", [HANDLES[0], HANDLES[9], HANDLES[-3], HANDLES[-2], HANDLES[-1]],
                         ids=["lane_v0", "mma_12_v7", "cta_v9", "cta_runtime", "dense"])
def test_exactness(env, name, kw, dims):
    gar, _, torch = env
    s, _ = lq_gpu.setup(env, kw, dims, seed=5)
    primal = lq_gpu.primal(env, s)
    cot = lq_gpu.cotangent(env, s, 2)
    base = lq_gpu.grad_bufs(env, s)
    s.adjoint(primal, cot, base, MU)
    base = lq_gpu.to_np(base)
    # zero cotangents: all-zero gradients
    zero = lq_gpu.grad_bufs(env, s)
    s.adjoint(primal, {k: torch.zeros_like(v) for k, v in cot.items()}, zero, MU)
    for k, v in lq_gpu.to_np(zero).items():
        assert np.all(v == 0.0), (name, "zero", k)
    # cotangents scaled by 2^k: gradients exactly 2^k times as large
    for e in (-40, 7, 40):
        g = lq_gpu.grad_bufs(env, s)
        s.adjoint(primal, {k: v * 2.0 ** e for k, v in cot.items()}, g, MU)
        for k, v in lq_gpu.to_np(g).items():
            assert np.array_equal(v, base[k] * 2.0 ** e), (name, e, k)
    # NULL cotangent fields: the same bits as explicit zero arrays
    for drop in (("vs", "lam0"), ("xs",), ("us", "vsT", "lams")):
        part = {k: (None if k in drop else v) for k, v in cot.items()}
        expl = {k: (torch.zeros_like(v) if k in drop else v) for k, v in cot.items()}
        a, b = lq_gpu.grad_bufs(env, s), lq_gpu.grad_bufs(env, s)
        s.adjoint(primal, part, a, MU)
        s.adjoint(primal, expl, b, MU)
        for k in GRADS:
            assert np.array_equal(lq_gpu.to_np(a)[k], lq_gpu.to_np(b)[k]), (name, drop, k)
    # NULL gradient outputs are not written; the requested ones are as in the full call
    for want in (("stage",), ("term", "g0"), ("G0",)):
        bufs = lq_gpu.grad_bufs(env, s)
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
    s, _ = lq_gpu.setup(env, kw, dims, seed=9)
    mu_b = np.array([MUS[b % 3] for b in range(B)])
    cot = lq_gpu.cotangent(env, s, 3)
    want = {k: np.empty(v.shape) for k, v in lq_gpu.grad_bufs(env, s).items()}
    want_out = {}
    for v in MUS:
        s.sweep(v)
        primal = lq_gpu.primal(env, s)
        g = lq_gpu.grad_bufs(env, s)
        s.adjoint(primal, cot, g, v)
        sel = mu_b == v
        for k, a in lq_gpu.to_np(g).items():
            want[k][sel] = a[sel]
        for k, a in lq_gpu.outputs(gar, s).items():
            want_out.setdefault(k, np.empty_like(a))[sel] = a[sel]
    for mu_arg in (mu_b, torch.tensor(mu_b, device="cuda")):
        s.sweep(mu_arg)
        primal = lq_gpu.primal(env, s)
        g = lq_gpu.grad_bufs(env, s)
        n0 = s.launch_count()
        s.adjoint(primal, cot, g, mu_arg)
        s.synchronize()
        assert s.launch_count() - n0 == 3
        for k, a in lq_gpu.to_np(g).items():
            assert np.array_equal(a, want[k]), (name, type(mu_arg), k)
        got_out = lq_gpu.outputs(gar, s)
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
    s, recs = lq_gpu.setup(env, kw, dims, seed=13)
    new_last = np.ascontiguousarray(gar.pack_problems(gen.generate_batch(99, B, 1, nx, nu, nc, nct))[0].reshape(B, -1))
    s.cycle_append(new_last)
    s.sweep(MU)
    primal = lq_gpu.primal(env, s)
    cot = lq_gpu.cotangent(env, s, 4)
    g = lq_gpu.grad_bufs(env, s)
    s.adjoint(primal, cot, g, MU)
    got, got_out = lq_gpu.to_np(g), lq_gpu.outputs(gar, s)
    rot = np.ascontiguousarray(np.concatenate([recs[0].reshape(B, N, -1)[:, 1:], new_last[:, None]], axis=1))
    f = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
    f.set_problem(rot, recs[1], recs[2], recs[3])
    f.sweep(MU)
    primal_f = lq_gpu.primal(env, f)
    for k in KEYS:
        assert torch.equal(primal_f[k], primal[k]), (name, k)
    gf = lq_gpu.grad_bufs(env, f)
    f.adjoint(primal_f, cot, gf, MU)
    for k, a in lq_gpu.to_np(gf).items():
        assert np.array_equal(got[k], a), (name, k)
    for k, a in lq_gpu.outputs(gar, f).items():
        assert np.array_equal(got_out[k], a, equal_nan=True), (name, k)
    s.close()
    f.close()


def _rc(gar, s, primal, cot, grad, mu=MU):
    pr = gar._fill(gar.LsIterate(), gar._LS_KEYS, primal)
    ct = gar._fill(gar.LsIterate(), gar._LS_KEYS, cot)
    gr = gar._fill(gar.LqGrad(), gar._GRAD_KEYS, grad)
    return gar.lib().ab2_gar_adjoint(s.h, C.c_double(mu), C.byref(pr), C.byref(ct), C.byref(gr), None)


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
        z = lq_gpu.zeros_like_outputs(env, s)
        assert _rc(gar, s, z, z, lq_gpu.grad_bufs(env, s)) == 2, kw  # AB2_ERR_UNSUPPORTED
        with pytest.raises(gar.GarError):
            s.adjoint(z, z, lq_gpu.grad_bufs(env, s), MU)
        assert s.launch_count() == n0
        s.close()
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    z = lq_gpu.zeros_like_outputs(env, s)
    assert _rc(gar, s, z, z, lq_gpu.grad_bufs(env, s)) == 4  # AB2_ERR_STATE: no problem set
    assert s.launch_count() == 0
    probs = gen.generate_batch(1, B, N, nx, nu, nc, nct)
    s.set_problem(*gar.pack_problems(probs))
    s.sweep(MU)
    s.synchronize()
    n0 = s.launch_count()
    alias = dict(z)
    alias["xs"] = s.device_ptr(gar.OUT_XS)  # the primal would be overwritten by the adjoint sweep
    assert _rc(gar, s, alias, z, lq_gpu.grad_bufs(env, s)) == 1
    inner = dict(z)
    inner["lams"] = s.device_ptr(gar.OUT_LBDAS) + 8 * nx  # overlapping, not at the start
    assert _rc(gar, s, inner, z, lq_gpu.grad_bufs(env, s)) == 1
    missing = dict(z)
    missing["us"] = None
    assert _rc(gar, s, missing, z, lq_gpu.grad_bufs(env, s)) == 1
    assert _rc(gar, s, z, z, lq_gpu.grad_bufs(env, s), mu=0.0) == 1  # constraints need mu > 0
    assert s.launch_count() == n0
    s.close()


@pytest.mark.parametrize("dims,kw", [((4, 2, 2, 1, 4, 3, 2), {}), ((7, 3, 2, 1, 7, 2, 2), {})],
                         ids=["warp", "cta_runtime"])
def test_gradcheck_lq_solve(env, dims, kw):
    gar, ag, torch = env
    nx, nu, nc, nct, nc0, N, B = dims
    probs = gen.generate_batch(21, B, N, nx, nu, nc, nct)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
    blocks, term, init = lq_gpu.block_inputs(torch, probs)
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
    primal = lq_gpu.primal(env, s)
    cot = lq_gpu.cotangent(env, s, 5)
    grad = lq_gpu.grad_bufs(env, s)
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
