"""Higher derivatives of the LQ solve on the GPU: the generalised streaming kernels (ab2_gar_rho_many,
ab2_gar_grad_many) against their numpy restatement, their bits against adjoint_many / tangent_many, independence of
nrhs and position, the handle's state, errors; lq_solve_higher's first derivatives bit for bit against lq_solve's, its
Hessian-vector product at DESIGN section 5's bar against extended-precision central differences of the gradient records
(tests/hp_higher_order.py), and one full-size HVP batch."""
import ctypes as C
import functools

import numpy as np
import pytest

import gen
import hp_higher_order as hho
import hp_reference as hp
import lq_adjoint_ref as aref
import lq_gpu
from lq_cases import check_bar, symmetric_dot
from lq_gpu import SERIAL
from lq_higher_ref import grad_modes, rho_modes

pytestmark = pytest.mark.gpu
KEYS = aref.KEYS
RECS = ("stage", "term", "G0", "g0")
MU = 1e-2
NRHS = 35  # past the gradient kernel's chunk of 16 and resolve's 32
# warp kernels (compile-time shapes, a record longer than one 512-double tile), the CTA kernels
# and C5 (nx 57, a 10 616-double record: the generalised gradient kernel stages one direction per chunk)
CASES = [h for h in SERIAL if h[0] in ("lane_v0", "lane_12_6_6", "mma_14_v6", "cta_v9", "cta_runtime")] + [
    ("c5", {}, (57, 28, 0, 0, 57, 1, 2))]
IDS = [h[0] for h in CASES]
# (a1 / z1 per direction, a2 / z2 per direction): the second term's vector per direction reloads the staged vectors
MODES = [(True, False), (True, True), (False, True)]
MODE_IDS = ["each1", "each12", "each2"]


@pytest.fixture(scope="module")
def env():
    return lq_gpu.gpu_env()


def _rel(got, want):
    return max(gen.rel_fro(got[k], want[k]) for k in want if np.asarray(want[k]).size)


def _d6(s):
    d = s.dims
    return d.nx, d.nu, d.nc, d.nct, d.nc0, d.horizon


def _shared(env, primal, seed):
    return {k: v[0] for k, v in lq_gpu.cots(env, None, primal, 1, seed).items()}


@pytest.mark.parametrize("each1,each2", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("name,kw,dims", CASES, ids=IDS)
def test_kernels_against_numpy_and_bits(env, name, kw, dims, each1, each2):
    gar, _, torch = env
    s, _ = lq_gpu.setup(env, kw, dims, 5, MU)
    d6, primal = _d6(s), lq_gpu.primal(env, s)
    before, epoch, launches = lq_gpu.outputs(gar, s), s.factor_epoch(), s.launch_count()
    dot1, dot2 = lq_gpu.dots(env, s, NRHS, 11), lq_gpu.dots(env, s, NRHS, 21)
    e, y1, y2 = (lq_gpu.cots(env, s, primal, NRHS, seed) for seed in (41, 51, 61))
    a1 = lq_gpu.cots(env, s, primal, NRHS, 31) if each1 else _shared(env, primal, 31)
    a2 = lq_gpu.cots(env, s, primal, NRHS, 71) if each2 else _shared(env, primal, 71)
    vecs = lambda d, each: lq_gpu.to_np(d) if each else lq_gpu.to_np(d) | {"each": False}
    pick = lambda d, each, j: {k: v[j:j + 1] for k, v in d.items()} if each else d
    for vec in (True, False):
        out = lq_gpu.sol_bufs(env, primal, NRHS)
        s.rho_many(dot1, a1, out, vec, dot2, a2, e)
        want = rho_modes(NRHS, d6, lq_gpu.to_np(dot1), vecs(a1, each1), vec, lq_gpu.to_np(dot2), vecs(a2, each2), lq_gpu.to_np(e))
        assert _rel(lq_gpu.to_np(out), want) <= 1e-12, vec
        grad = lq_gpu.grad_bufs_many(env, s, NRHS)
        s.grad_many(y1, a1, grad, vec, y2, a2)
        want = grad_modes(NRHS, d6, lq_gpu.to_np(y1), vecs(a1, each1), vec, lq_gpu.to_np(y2), vecs(a2, each2))
        assert _rel(lq_gpu.to_np(grad), want) <= 1e-12, vec
        # right-hand side j alone gives the bits it had among NRHS
        for j in (0, 17, NRHS - 1):
            one = lq_gpu.sol_bufs(env, primal, 1)
            s.rho_many({k: v[j:j + 1] for k, v in dot1.items()}, pick(a1, each1, j), one, vec,
                       {k: v[j:j + 1] for k, v in dot2.items()}, pick(a2, each2, j),
                       {k: v[j:j + 1] for k, v in e.items()})
            assert all(torch.equal(one[k][0], out[k][j]) for k in KEYS), (vec, j)
            g1 = lq_gpu.grad_bufs_many(env, s, 1)
            s.grad_many({k: v[j:j + 1] for k, v in y1.items()}, pick(a1, each1, j), g1, vec,
                        {k: v[j:j + 1] for k, v in y2.items()}, pick(a2, each2, j))
            assert all(torch.equal(g1[k][0], grad[k][j]) for k in RECS), (vec, j)
    if (each1, each2) != MODES[0]:
        s.close()
        return
    # one term with the vector blocks and a shared primal: tangent_many's work and adjoint_many's gradient, bit for bit;
    # the same primal given per direction runs the generalised instantiation and gives the same bits
    work, zd = lq_gpu.sol_bufs(env, primal, NRHS), lq_gpu.sol_bufs(env, primal, NRHS)
    s.tangent_many(primal, dot1, work, zd, MU)
    rho, rho_each = lq_gpu.sol_bufs(env, primal, NRHS), lq_gpu.sol_bufs(env, primal, NRHS)
    s.rho_many(dot1, primal, rho)
    s.rho_many(dot1, {k: v.expand(NRHS, *v.shape).contiguous() for k, v in primal.items()}, rho_each)
    assert all(torch.equal(rho[k], work[k]) and torch.equal(rho_each[k], work[k]) for k in KEYS)
    y, g_adj = lq_gpu.sol_bufs(env, primal, NRHS), lq_gpu.grad_bufs_many(env, s, NRHS)
    s.adjoint_many(primal, y1, y, g_adj, MU)
    g, g_each = lq_gpu.grad_bufs_many(env, s, NRHS), lq_gpu.grad_bufs_many(env, s, NRHS)
    s.grad_many(y, primal, g)
    s.grad_many(y, {k: v.expand(NRHS, *v.shape).contiguous() for k, v in primal.items()}, g_each)
    assert all(torch.equal(g[k], g_adj[k]) and torch.equal(g_each[k], g_adj[k]) for k in RECS)
    # the calls read and write nothing of the handle's
    after = lq_gpu.outputs(gar, s)
    assert all(np.array_equal(before[k], after[k]) for k in before) and s.factor_epoch() == epoch
    assert s.launch_count() > launches
    s.close()


def test_errors_launch_nothing(env):
    gar, _, torch = env
    s, _ = lq_gpu.setup(env, {}, (4, 2, 2, 2, 4, 6, 9), 3, MU)
    primal = lq_gpu.primal(env, s)
    dot, a = lq_gpu.dots(env, s, 2, 1), lq_gpu.cots(env, s, primal, 2, 2)
    out, grad = lq_gpu.sol_bufs(env, primal, 2), lq_gpu.grad_bufs_many(env, s, 2)
    n0 = s.launch_count()
    fill = lambda d, T: C.byref(gar._fill(T(), [f for f, _ in T._fields_], d))
    assert gar.lib().ab2_gar_rho_many(s.h, -1, 1, fill(dot, gar.LqTangent), fill(a, gar.LsIterate), 1, None, None, 0,
                                      None, fill(out, gar.LsIterate), None) != 0  # nrhs < 0
    with pytest.raises(gar.GarError, match="overlaps"):  # out on top of the tangent records
        s.rho_many(dot, a, {k: dot["stage"].view(-1)[:v.numel()].view(v.shape) for k, v in out.items()})
    with pytest.raises(gar.GarError, match="overlaps"):  # a gradient record on top of y
        s.grad_many(a, primal, {"G0": a["xs"].view(-1)[:grad["G0"].numel()].view(grad["G0"].shape)})
    with pytest.raises(gar.GarError, match="NULL"):
        s.rho_many(dot, {k: (None if k == "us" else v) for k, v in a.items()}, out)
    assert s.launch_count() == n0
    p = gar.CudaRiccatiBatch(4, 2, 2, 2, 4, 6, 9, nth=2)
    with pytest.raises(gar.GarError, match="parametric"):
        p.grad_many(a, primal, grad)
    p.close()
    s.close()


def _torch_recs(env, s, recs):
    torch = env[2]
    return [torch.tensor(np.ascontiguousarray(a), device="cuda").reshape(sh)
            for a, sh in zip(recs, lq_gpu.rec_shapes(s).values())]


@pytest.mark.parametrize("kw", [{}, dict(variant=9)], ids=["warp", "cta_v9"])
def test_first_derivatives_bit_equal_lq_solve(env, kw):
    _, ag, torch = env
    s, recs = lq_gpu.setup(env, kw, (4, 2, 2, 2, 4, 5, 6), 7, MU)
    P = _torch_recs(env, s, recs)
    for k in (0, 1, 5):
        for i in (0, 1, 2, 3):
            f = lambda lq: (lambda x: lq(s, *[x if n == i else r for n, r in enumerate(P)], MU)[k])
            for J in (torch.func.jacrev, torch.func.jacfwd):
                assert torch.equal(J(f(ag.lq_solve_higher))(P[i]), J(f(ag.lq_solve))(P[i])), (k, i, J.__name__)
    outs_h, outs = ag.lq_solve_higher(s, *P, MU), ag.lq_solve(s, *P, MU)
    assert all(torch.equal(a, b) for a, b in zip(outs_h, outs))
    s.close()


def _loss(torch, W):
    return lambda outs: sum((w * o).sum() + 0.5 * (w * o * o).sum() for w, o in zip(W, outs))


# name: ((nx, nu, nc, nct, nc0, N), batch, mu)
HVP_CASES = {
    "c3_mu1e-3": ((4, 2, 2, 0, 4, 6), 3, 1e-3),
    "c3_nct2_mu1e-8": ((4, 2, 2, 2, 4, 5), 2, 1e-8),
    "c2": ((12, 6, 0, 0, 12, 5), 2, 1e-8),
}
HVP_ITEMS = [(n, kw) for n in HVP_CASES for kw in ({}, dict(variant=9))]
HVP_DIRECTIONS = 2


@functools.lru_cache(maxsize=None)
def hvp_case(name):
    """The problems, the loss weights, the directions, and per direction the extended-precision HVP and e_ref."""
    d6, B, mu = HVP_CASES[name]
    nx, nu, nc, nct, nc0, N = d6
    probs = gen.general_initial_condition(gen.generate_batch(8000 + sum(map(ord, name)), B, N, nx, nu, nc, nct), nc0, 8)
    recs = hp.records(probs)
    rng = np.random.default_rng(3)
    W = {k: rng.standard_normal(sh) for k, sh in aref._shapes(d6, B).items()}
    dots = [symmetric_dot(rng, d6, B) for _ in range(HVP_DIRECTIONS)]
    refs = [hho.hvp_hp(probs, mu, W, dot) for dot in dots]
    e_refs = [hp.grad_errors(hho.hvp_fp64(recs, d6, mu, W, dot), ref, d6) for dot, ref in zip(dots, refs)]
    return recs, W, dots, refs, e_refs


@pytest.mark.parametrize("name,kw", HVP_ITEMS, ids=["%s-%s" % (n, "cta_v9" if kw else "warp") for n, kw in HVP_ITEMS])
def test_hvp_meets_the_bar(env, name, kw):
    """A batch of HVPs (vmap over directions of jvp of grad, with respect to all four inputs) at DESIGN section 5's
    bar: e_kernel <= max(16 e_ref, 64 u) per record block, against the extended-precision central differences of the
    gradient records, e_ref the fp64 composition's error on the oracle's solves."""
    gar, ag, torch = env
    d6, B, mu = HVP_CASES[name]
    recs, W, dots, refs, e_refs = hvp_case(name)
    s = gar.CudaRiccatiBatch(*d6, B, **kw)
    s.set_problem(*[np.ascontiguousarray(a) for a in recs])
    P = _torch_recs(env, s, recs)
    Wt = [torch.tensor(W[k], device="cuda") for k in KEYS]
    dirs = [torch.stack([torch.tensor(d[k], device="cuda") for d in dots]) for k in RECS]
    f = lambda *x: _loss(torch, Wt)(ag.lq_solve_higher(s, *x, mu))
    hv = torch.func.vmap(lambda *v: torch.func.jvp(torch.func.grad(f, argnums=(0, 1, 2, 3)), tuple(P), v)[1])(*dirs)
    for j in range(HVP_DIRECTIONS):
        e = hp.grad_errors({k: h[j].cpu().numpy() for k, h in zip(RECS, hv)}, refs[j], d6)
        title = "%s %s HVP direction %d" % (name, "cta_v9" if kw else "warp", j)
        print("\n" + hp.table(title, e_refs[j], e))
        check_bar(e, e_refs[j], title)
    s.close()


def test_full_size_hvp(env):
    """One HVP batch at C2 (B 4096, V 8): finite, and equal to the fp64 composition on the oracle's solves on
    instances sampled across the launch."""
    _, ag, torch = env
    dims, mu, V = (12, 6, 0, 0, 12, 100, 4096), 1e-2, 8
    s, recs = lq_gpu.setup(env, {}, dims, 2, mu)
    P = _torch_recs(env, s, recs)
    outs = ag.lq_solve(s, *P, mu)
    g = torch.Generator(device="cuda").manual_seed(6)
    W = [torch.randn(o.shape, generator=g, dtype=torch.float64, device="cuda") for o in outs]
    dirs = torch.randn((V,) + tuple(P[1].shape), generator=g, dtype=torch.float64, device="cuda")  # along term
    f = lambda st, tm: _loss(torch, W)(ag.lq_solve_higher(s, st, tm, P[2], P[3], mu))
    hv = torch.func.vmap(lambda v: torch.func.jvp(torch.func.grad(f, argnums=(0, 1)), (P[0], P[1]),
                                                  (torch.zeros_like(P[0]), v))[1])(dirs)
    assert all(bool(torch.isfinite(h).all()) for h in hv)
    idx = np.array([0, dims[6] // 2, dims[6] - 1])
    sub = [np.ascontiguousarray(r[idx]) for r in recs]
    Wn = {k: w[idx].cpu().numpy() for k, w in zip(KEYS, W)}
    for j in (0, V - 1):
        dot = dict(term=dirs[j][idx].cpu().numpy())
        want = hho.hvp_fp64(sub, dims[:6], mu, Wn, dot)
        got = {k: h[j][idx].cpu().numpy() for k, h in zip(("stage", "term"), hv)}
        assert _rel(got, {k: want[k] for k in ("stage", "term")}) <= 1e-10, j
    s.close()
