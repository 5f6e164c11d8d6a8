"""Iterative refinement of the batched LQ solve on the GPU (ab2_gar_refine, ab2_gar_refine_many, gar.h): accuracy
against the extended-precision solve, residual norms against ab2_gar_kkt_error, the handle's other outputs untouched,
refine_many on resolve outputs with bit-exact independence of nrhs, the per-instance-mu twins, state rules and errors,
and full-size batches."""
import ctypes as C

import numpy as np
import pytest

import gen
import hp_reference as hp
import lq_adjoint_ref as aref
import lq_refine_ref as fref
import lq_resolve_ref as rref
import lq_gpu
from lq_cases import batch_records, errors, refine_case, refined_on_oracle
from lq_gpu import HANDLES

pytestmark = pytest.mark.gpu
# every kernel kind resolve serves: warp variants (packed Vxx), the CTA kernel, a run-time shape, C5 dims
KINDS = [h for h in HANDLES if not h[1].get("dense")] + [("c5_dims", {}, (57, 28, 0, 0, 57, 3, 2))]
KIND_IDS = [h[0] for h in KINDS]


@pytest.fixture(scope="module")
def env():
    return lq_gpu.gpu_env()


def _slack(z):
    """Rounding of a residual evaluation: two correct fp64 evaluations of max |K z + h| differ by about this much."""
    return 1e-13 * max(1.0, max(float(np.abs(np.asarray(v)).max(initial=0.0)) for v in z.values()))


def _not_worse(after, before, z):
    return np.all(after <= before + _slack(z))


def _traj(gar, s):
    return {k: s.get(w).copy() for k, w in zip(rref.SOL, (gar.OUT_XS, gar.OUT_US, gar.OUT_VS, gar.OUT_VST,
                                                          gar.OUT_LBD0, gar.OUT_LBDAS))}


def _handle(env, kw, dims, seed, mu, probs=None):
    gar, _, _ = env
    nx, nu, nc, nct, nc0, N, B = dims
    if probs is None:
        probs = gen.generate_batch(seed, B, N, nx, nu, nc, nct)
    recs = [np.ascontiguousarray(a) for a in gar.pack_problems(probs)]
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
    s.set_problem(*recs)
    s.sweep(mu)
    return s, recs


def _dev(env, h):
    _, _, torch = env
    return {k: torch.tensor(np.ascontiguousarray(v), device="cuda") for k, v in h.items()}


def _sol(env, d6, B, nrhs, fill=float("nan")):
    _, _, torch = env
    return {k: torch.full((nrhs,) + s, fill, dtype=torch.float64, device="cuda")
            for k, s in zip(rref.SOL, rref.rhs_shapes(d6, B).values())}


def _work(env, d6, B, nrhs):
    _, _, torch = env
    shapes = rref.rhs_shapes(d6, B)
    w = {k: torch.full((nrhs,) + s, float("nan"), dtype=torch.float64, device="cuda") for k, s in shapes.items()}
    w.update(_sol(env, d6, B, nrhs))
    return w


@pytest.mark.parametrize("name", ["c3_mu1e-8", "c3_mu1e-11", "c3_nct_mu1e-8", "pivots_2x2_mu1e-8", "interchanges"])
def test_refined_device_trajectory_meets_the_bar(env, name):
    """After refine(2) every trajectory family is within max(16 e_ref, 64 u) of the extended-precision solve, e_ref the
    refined CPU restatement's error; the last residual norm is not above the first."""
    gar, _, _ = env
    probs, recs, case, mu = refine_case(name)
    nx, nu, nc, nct, nc0, N = case
    B = len(probs)
    zc, _, _, want, _ = refined_on_oracle(probs, recs, case, mu)
    e_ref = errors(zc, want, case)
    s, _ = _handle(env, {}, case + (B,), 0, mu, probs=probs)
    z0 = _traj(gar, s)
    norms = s.refine(mu, 2, norms=True)
    z = _traj(gar, s)
    e = errors({k: v[None] for k, v in z.items()}, want, case)
    bad = {f: (e[f], e_ref[f]) for f in e if not e[f] <= max(16 * e_ref[f], hp.FLOOR)}
    assert not bad, (name, bad)
    assert _not_worse(norms[:, -1], norms[:, 0], z), norms
    if name == "c3_mu1e-11":  # the unrefined device trajectory misses 64 u
        assert max(errors({k: v[None] for k, v in z0.items()}, want, case).values()) > hp.FLOOR
    s.close()


@pytest.mark.parametrize("name,kw,dims", KINDS, ids=KIND_IDS)
def test_norms_state_and_kernel_kinds(env, name, kw, dims):
    gar, _, torch = env
    nx, nu, nc, nct, nc0, N, B = dims
    mu = 1e-5
    s, recs = _handle(env, kw, dims, 31, mu)
    before = lq_gpu.outputs(gar, s)
    e0 = s.factor_epoch()
    # steps = 0: the first norm only, the trajectory bit-identical; it equals max(kkt_error) within rounding
    z0 = _traj(gar, s)
    n0 = s.refine(mu, 0, norms=True)
    k0 = s.kkt_error(mu).max(axis=1)
    assert n0.shape == (B, 1)
    assert np.allclose(n0[:, 0], k0, rtol=0, atol=_slack(z0)), (n0[:, 0], k0)
    after0 = lq_gpu.outputs(gar, s)
    for k, a in before.items():
        assert np.array_equal(a, after0[k], equal_nan=True), (name, k)
    # two steps: the first column repeats, the last equals the kkt error of the refined trajectory
    norms = s.refine(mu, 2, norms=True)
    z = _traj(gar, s)
    assert np.array_equal(norms[:, 0], n0[:, 0])
    assert np.allclose(norms[:, -1], s.kkt_error(mu).max(axis=1), rtol=0, atol=_slack(z))
    assert _not_worse(norms[:, -1], norms[:, 0], z), norms
    # every other output bit-identical, the epoch unchanged; the refined trajectory is close to the unrefined one
    after = lq_gpu.outputs(gar, s)
    for k, a in before.items():
        if k not in range(gar.OUT_XS, gar.OUT_LBDAS + 1):
            assert np.array_equal(a, after[k], equal_nan=True), (name, k)
    assert s.factor_epoch() == e0
    for k in rref.SOL:
        assert gen.rel_fro(z[k], z0[k]) <= 1e-8, (name, k)
    s.close()


@pytest.mark.parametrize("dims,general_g0", [((12, 6, 0, 0, 12, 20, 64), False), ((4, 2, 2, 2, 3, 20, 96), True),
                                             ((57, 28, 0, 0, 57, 6, 4), False)], ids=["C2", "C3_nct_G0", "C5"])
def test_kkt_error_is_the_residual_norm(env, dims, general_g0):
    """kkt_error's three norms are the per-family maxima of refine's residual: their maximum equals refine's first norm
    bit for bit, with a scalar and a per-instance mu, on a fresh handle and after cycle_append and a sweep (nonzero ring
    head).  A NaN in one instance's x makes that instance's dynamics and stationarity norms NaN and leaves every other
    instance's norms as they were."""
    gar, _, torch = env
    nx, nu, nc, nct, nc0, N, B = dims
    probs = gen.generate_batch(81, B, N, nx, nu, nc, nct)
    if general_g0:
        gen.general_initial_condition(probs, nc0, 82)
    _, srec = aref.stage_offsets(nx, nu, nc)
    new_last = np.zeros((B, srec))
    new_last[:, :gen.stage_record(probs[0].stages[1]).size] = [gen.stage_record(p.stages[1]) for p in probs]
    for mu in (1e-6, np.geomspace(1e-8, 1e-4, B)):
        s, _ = _handle(env, {}, dims, 0, mu, probs=probs)
        for ring in (False, True):
            if ring:
                s.cycle_append(new_last)
                s.sweep(mu)
            k = s.kkt_error(mu)
            n = s.refine(mu, 0, norms=True)[:, 0]
            assert np.all(np.isfinite(k)) and np.any(k > 0)
            assert np.array_equal(k.max(axis=1).view(np.uint64), n.view(np.uint64)), (ring, k.max(axis=1), n)
        xs = torch.as_tensor(lq_gpu.DeviceArray(s.device_ptr(gar.OUT_XS), B * (N + 1) * nx), device="cuda")
        xs[(1 * (N + 1) + N // 2) * nx] = float("nan")  # instance 1, knot N / 2, x[0]
        torch.cuda.synchronize()
        kn = s.kkt_error(mu)
        assert np.isnan(kn[1, 0]) and np.isnan(kn[1, 2]), kn[1]
        others = np.arange(B) != 1
        assert np.array_equal(kn[others].view(np.uint64), k[others].view(np.uint64))
        s.close()


@pytest.mark.parametrize("name,kw,dims", [KINDS[i] for i in (0, 8, 16, 17, 18)],
                         ids=[KIND_IDS[i] for i in (0, 8, 16, 17, 18)])
def test_refine_many(env, name, kw, dims):
    gar, _, torch = env
    nx, nu, nc, nct, nc0, N, B = dims
    d6 = dims[:6]
    mu = 1e-8
    s, recs = _handle(env, kw, dims, 41, mu)
    nrhs = 32
    h = _dev(env, rref.random_rhs(np.random.default_rng(42), d6, B, nrhs))
    z0 = _sol(env, d6, B, nrhs)
    s.resolve(h, z0, mu)
    # one step: work holds the dense residual of the input and its correction
    z = {k: v.clone() for k, v in z0.items()}
    w = _work(env, d6, B, nrhs)
    s.refine_many(h, z, w, mu, steps=1)
    st = recs[0].reshape(B, N, -1)
    G0, g0 = recs[2].reshape(B, -1), recs[3].reshape(B, -1)
    zn = {k: v.cpu().numpy() for k, v in z0.items()}
    r = fref.residual(st, recs[1], G0, g0, zn, {k: v.cpu().numpy() for k, v in h.items()}, d6, mu)
    scale = (max(float(v.abs().max()) for v in h.values() if v.numel())
             + 10 * max(float(v.abs().max()) for v in z0.values() if v.numel()))
    for k in rref.RHS:
        assert np.abs(w[k].cpu().numpy() - r[k]).max(initial=0.0) <= 1e-13 * scale, (name, k)
    for k in rref.SOL:
        assert torch.equal(z[k], z0[k] + w[k]), (name, k)
    # two steps with norms on the device; bit-identical for nrhs 1, 3 and 32 and across positions
    z32 = {k: v.clone() for k, v in z0.items()}
    n32 = torch.zeros((nrhs, B, 3), dtype=torch.float64, device="cuda")
    s.refine_many(h, z32, _work(env, d6, B, nrhs), mu, steps=2, norms=n32)
    for lo, hi in ((0, 1), (5, 8), (31, 32)):
        zz = {k: v[lo:hi].clone() for k, v in z0.items()}
        nn = s.refine_many({k: v[lo:hi].contiguous() for k, v in h.items()}, zz, _work(env, d6, B, hi - lo), mu,
                           steps=2, norms=True)
        for k in rref.SOL:
            assert torch.equal(zz[k], z32[k][lo:hi]), (name, lo, k)
        assert np.array_equal(nn, n32[lo:hi].cpu().numpy()), (name, lo)
    # each refined right-hand side is still the solution of its replaced problem, and the norm has not grown
    n = n32.cpu().numpy()
    assert _not_worse(n[..., -1], n[..., 0], zn), name
    for k in rref.SOL:
        assert gen.rel_fro(z32[k].cpu().numpy(), zn[k]) <= 1e-4, (name, k)
    # NULL rhs fields are zero
    part = {k: (v if k in ("q", "g0") else None) for k, v in h.items()}
    za, zb = ({k: v.clone() for k, v in z0.items()} for _ in range(2))
    s.refine_many(part, za, _work(env, d6, B, nrhs), mu, steps=1)
    s.refine_many({k: (v if v is not None else torch.zeros_like(h[k])) for k, v in part.items()}, zb,
                  _work(env, d6, B, nrhs), mu, steps=1)
    for k in rref.SOL:
        assert torch.equal(za[k], zb[k]), k
    s.close()


@pytest.mark.parametrize("name", ["c3_mu1e-11", "c3_nct_mu1e-8"])
def test_refine_many_on_resolve_outputs_meets_the_bar(env, name):
    """Right-hand sides resolved at small mu, refined twice: each within max(16 e_ref, 64 u) of the extended-precision
    solve of its replaced problem, e_ref the CPU restatement refined the same way on the oracle's factorisation."""
    gar, _, _ = env
    probs, recs, case, mu = refine_case(name)
    B = len(probs)
    s, _ = _handle(env, {}, case + (B,), 0, mu, probs=probs)
    h = rref.random_rhs(np.random.default_rng(len(name)), case, B, 2)
    hd = _dev(env, h)
    z = _sol(env, case, B, 2)
    s.resolve(hd, z, mu)
    s.refine_many(hd, z, _work(env, case, B, 2), mu, steps=2)
    for j in range(2):
        rp = rref.replaced_problems(probs, {k: v[j] for k, v in h.items()})
        rr = [np.ascontiguousarray(a) for a in batch_records(rp, case)]
        zc, _, _, want, _ = refined_on_oracle(rp, rr, case, mu)
        e_ref = errors(zc, want, case)
        e = errors({k: v[j:j + 1].cpu().numpy() for k, v in z.items()}, want, case)
        bad = {f: (e[f], e_ref[f]) for f in e if not e[f] <= max(16 * e_ref[f], hp.FLOOR)}
        assert not bad, (name, j, bad)
    s.close()


def test_v_twins(env):
    gar, _, torch = env
    dims = (4, 2, 2, 2, 4, 6, 6)
    nx, nu, nc, nct, nc0, N, B = dims
    d6 = dims[:6]
    mus = np.array([1e-3, 1e-3, 1e-8, 1e-8, 1e-5, 1e-5])
    probs = gen.generate_batch(51, B, N, nx, nu, nc, nct)
    s, recs = _handle(env, {}, dims, 0, mus, probs=probs)
    nv = s.refine(mus, 2, norms=True)
    zv = _traj(gar, s)
    sd, _ = _handle(env, {}, dims, 0, torch.tensor(mus, device="cuda"), probs=probs)
    nd = sd.refine(torch.tensor(mus, device="cuda"), 2, norms=True)
    assert np.array_equal(nv, nd)
    for k, v in _traj(gar, sd).items():
        assert np.array_equal(v, zv[k]), k
    h = _dev(env, rref.random_rhs(np.random.default_rng(52), d6, B, 3))
    zm = _sol(env, d6, B, 3)
    s.resolve(h, zm, mus)
    zmv = {k: v.clone() for k, v in zm.items()}
    nmv = s.refine_many(h, zmv, _work(env, d6, B, 3), mus, steps=2, norms=True)
    for m in (1e-3, 1e-8, 1e-5):  # each group of instances that share a mu equals the scalar calls
        idx = np.flatnonzero(mus == m)
        one, _ = _handle(env, {}, (nx, nu, nc, nct, nc0, N, len(idx)), 0, m, probs=[probs[i] for i in idx])
        ns = one.refine(m, 2, norms=True)
        assert np.array_equal(ns, nv[idx]), m
        for k, v in _traj(gar, one).items():
            assert np.array_equal(v, zv[k][idx]), (m, k)
        hs = {k: v[:, idx].contiguous() for k, v in h.items()}
        zs = _sol(env, d6, len(idx), 3)
        one.resolve(hs, zs, m)
        nms = one.refine_many(hs, zs, _work(env, d6, len(idx), 3), m, steps=2, norms=True)
        for k in rref.SOL:
            assert torch.equal(zs[k], zmv[k][:, idx]), (m, k)
        assert np.array_equal(nms, nmv[:, idx]), m
        one.close()
    s.close()
    sd.close()


def _rc(gar, s, mu, steps, norms=None):
    return gar.lib().ab2_gar_refine(s.h, C.c_double(mu), int(steps), norms, None)


def _rcm(gar, s, mu, nrhs, steps, rhs, z, work):
    rh = gar._fill(gar.LqRhs(), gar._RHS_KEYS, rhs)
    zz = gar._fill(gar.LsIterate(), gar._LS_KEYS, z)
    wk = gar._fill(gar.LqRefineWork(), gar._RHS_KEYS + gar._LS_KEYS, work)
    return gar.lib().ab2_gar_refine_many(s.h, C.c_double(mu), int(nrhs), int(steps), C.byref(rh), C.byref(zz),
                                         C.byref(wk), None, None)


def test_state_and_errors(env):
    gar, _, torch = env
    dims = (4, 2, 2, 2, 4, 6, 5)
    nx, nu, nc, nct, nc0, N, B = dims
    d6 = dims[:6]
    mu = 1e-2
    probs = gen.generate_batch(61, B, N, nx, nu, nc, nct)
    recs = gar.pack_problems(probs)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    z, w = _sol(env, d6, B, 2, 0.0), _work(env, d6, B, 2)
    assert _rc(gar, s, mu, 1) == 4 and _rcm(gar, s, mu, 2, 1, {}, z, w) == 4  # no problem
    s.set_problem(*recs)
    assert _rc(gar, s, mu, 1) == 4 and _rcm(gar, s, mu, 2, 1, {}, z, w) == 4  # no backward since set_problem
    s.backward(mu)
    assert _rc(gar, s, mu, 1) == 4  # a backward alone: no primal trajectory
    assert _rcm(gar, s, mu, 2, 1, {}, z, w) == 0  # refine_many needs only the factorisation
    s.forward()
    assert _rc(gar, s, mu, 1) == 0
    s.sweep(mu)
    primal = {k: torch.tensor(v, device="cuda") for k, v in _traj(gar, s).items()}
    s.adjoint(primal, {k: torch.ones_like(v) for k, v in primal.items()},
              dict(stage=torch.empty((B, N, s.srec), dtype=torch.float64, device="cuda")), mu)
    assert _rc(gar, s, mu, 1) == 4  # after an adjoint
    s.forward()
    assert _rc(gar, s, mu, 1) == 4  # a forward on the adjoint's factorisation is not the primal either
    s.sweep(mu)
    s.tangent(primal, {}, mu)
    assert _rc(gar, s, mu, 1) == 4  # after a tangent
    s.sweep(mu)
    s.synchronize()
    n0 = s.launch_count()
    assert _rc(gar, s, mu, -1) == 1
    assert _rc(gar, s, 0.0, 1) == 1
    assert _rcm(gar, s, mu, -1, 1, {}, z, w) == 1
    assert _rcm(gar, s, mu, 2, -1, {}, z, w) == 1
    assert _rcm(gar, s, 0.0, 2, 1, {}, z, w) == 1
    for k in rref.SOL:
        assert _rcm(gar, s, mu, 2, 1, {}, dict(z, **{k: None}), w) == 1, k
    for k in rref.RHS + rref.SOL:
        assert _rcm(gar, s, mu, 2, 1, {}, z, dict(w, **{k: None})) == 1, k
    assert _rcm(gar, s, mu, 2, 1, dict(q=z["xs"]), z, w) == 1          # rhs with z
    assert _rcm(gar, s, mu, 2, 1, dict(f=w["lams"]), z, w) == 1        # rhs with work
    assert _rcm(gar, s, mu, 2, 1, {}, dict(z, us=w["r"]), w) == 1      # z with work
    assert _rcm(gar, s, mu, 2, 1, {}, dict(z, vs=z["us"]), w) == 1     # z with itself
    assert _rcm(gar, s, mu, 2, 1, {}, z, dict(w, xs=w["q"])) == 1      # the two halves of work
    assert _rcm(gar, s, mu, 0, 1, {}, z, w) == 0                       # nrhs = 0
    assert _rc(gar, s, mu, 0) == 0                                     # steps = 0 without norms
    assert s.launch_count() == n0  # nothing launched on an error, for nrhs = 0 or for steps = 0 without norms
    assert _rc(gar, s, mu, 2) == 0
    assert s.launch_count() == n0 + 2 * 3
    s.refine(mu, 1, norms=True)
    assert s.launch_count() == n0 + 2 * 3 + 4
    # cycle_append without a backward
    _, srec = aref.stage_offsets(nx, nu, nc)
    nl = np.zeros((B, srec))
    rec = gen.stage_record(gen.generate_batch(9, 1, 1, nx, nu, nc, nct)[0].stages[0])
    nl[:, :rec.size] = rec
    s.cycle_append(nl)
    assert _rc(gar, s, mu, 1) == 4 and _rcm(gar, s, mu, 2, 1, {}, z, w) == 4
    s.sweep(mu)  # after the backward the records are read through the ring head
    norms = s.refine(mu, 2, norms=True)
    z = _traj(gar, s)
    assert np.allclose(norms[:, -1], s.kkt_error(mu).max(axis=1), rtol=0, atol=_slack(z))
    assert _not_worse(norms[:, -1], norms[:, 0], z)
    s.close()
    for kw in (dict(dense=True), dict(legs=2), dict(nth=2)):
        u = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
        assert _rc(gar, u, mu, 1) == 2 and _rcm(gar, u, mu, 2, 1, {}, z, w) == 2, kw
        u.close()


@pytest.mark.parametrize("dims,mu", [((12, 6, 0, 0, 12, 100, 4096), 1e-8), ((4, 2, 2, 2, 4, 100, 16384), 1e-8)],
                         ids=["C2", "C3"])
def test_full_size(env, dims, mu):
    """Every instance's refined KKT error is at most its unrefined one (up to the rounding of evaluating it)."""
    gar, _, _ = env
    s, _ = _handle(env, {}, dims, 71, mu)
    k0 = s.kkt_error(mu).max(axis=1)
    norms = s.refine(mu, 2, norms=True)
    k2 = s.kkt_error(mu).max(axis=1)
    z = _traj(gar, s)
    assert np.allclose(norms[:, 0], k0, rtol=0, atol=_slack(z))
    worse = np.flatnonzero(k2 > k0 + _slack(z))
    assert worse.size == 0, (worse[:10], k0[worse[:10]], k2[worse[:10]])
    print("C%s: max unrefined %.2e, max refined %.2e, instances improved %d of %d"
          % (dims, k0.max(), k2.max(), int((k2 < k0).sum()), k0.size))
    s.close()
