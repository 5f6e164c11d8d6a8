"""Derivatives of a parametric solution with respect to theta on the device: ab2_gar_theta_tangent (J d),
ab2_gar_theta_adjoint (J^T zbar) and autograd.lq_solve_theta.

Parity: the device results against the extended-precision Jacobian (lq_theta_ref.theta_jacobian) at the bar
e_kernel <= max(16 e_oracle, 64 u), e_oracle the fp64 restatement on the oracle's factors (tests/lq_theta_ref.py), on
batches of 2 grid + 3 instances (each its own problem) sampled on both sides of the CTA kernel's strides.  Also the
transposition and affine identities, bit-for-bit invariance, an untouched handle, every return code, and the torch
entry point in both modes and to second order."""
import ctypes as C
import functools

import numpy as np
import pytest

import hp_reference as hp
import lq_cases
import lq_gpu
import lq_theta_ref as tref

pytestmark = pytest.mark.gpu

INVALID, UNSUPPORTED, STATE = 1, 2, 4
KEYS = ("xs", "us", "vs", "vsT", "lam0", "lams")
FAC = ("fb", "fth", "Vxx", "Vxt", "kkt0fth", "fbT")


@pytest.fixture(scope="module")
def env():
    return lq_gpu.gpu_env()


# name: (nx, nu, nc, nct, nc0, nth, N, mueq): C2 and C3 dimensions, and nx 48 nu 24, the largest C5-like shape a
# parametric handle accepts (C5 itself, nx 57 nu 28, does not fit the CTA sweep with theta columns).  Short horizons:
# the reference runs at 50 digits.
CASES = {"c2_nth4": (12, 6, 0, 0, 12, 4, 6, 1e-8), "c2_nth12": (12, 6, 0, 0, 12, 12, 6, 1e-8),
         "c3_nth2": (4, 2, 2, 2, 4, 2, 20, 1e-3), "c5like_nth4": (48, 24, 0, 0, 48, 4, 2, 1e-8)}


def problems(name, B):
    nx, nu, nc, nct, nc0, nth, N, _ = CASES[name]
    return [lq_cases.make_problem([7100 + sum(map(ord, name)), b], N, nx, nu, nc, nct, nth, gv=True) for b in range(B)]


def handle(gar, name, B):
    nx, nu, nc, nct, nc0, nth, N, mueq = CASES[name]
    probs = problems(name, B)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, nth=nth)
    s.set_problem(*gar.pack_problems(probs))
    s.backward(mueq)
    thetas = np.random.default_rng(B).standard_normal((B, nth))
    s.forward(theta=thetas)
    assert np.all(s.status() == 0)
    return s, probs, thetas


@functools.lru_cache(maxsize=None)
def batch_of(name):
    """(B, sampled instances) with B = 2 grid + 3 of the CTA kernel for this shape."""
    import aligator_b200.gar as gar
    nx, nu, nc, nct, nc0, nth, N, _ = CASES[name]
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, 1 << 12, nth=nth)
    g = s.kernel_info()["grid"]
    s.close()
    B = 2 * g + 3
    return B, sorted({0, g, B - 1})


def sol(torch, d7, B, n):
    nx, nu, nc, nct, nc0, nth, N = d7
    shapes = dict(xs=(B, N + 1, nx), us=(B, N, nu), vs=(B, N, nc), vsT=(B, nct), lam0=(B, nc0), lams=(B, N, nx))
    return {k: torch.empty((n,) + s, dtype=torch.float64, device="cuda") for k, s in shapes.items()}


def d7_of(name):
    nx, nu, nc, nct, nc0, nth, N, _ = CASES[name]
    return nx, nu, nc, nct, nc0, nth, N


@pytest.mark.parametrize("name", list(CASES))
def test_parity_against_extended_precision(env, name):
    gar, _, torch = env
    nx, nu, nc, nct, nc0, nth, N, mueq = CASES[name]
    B, idx = batch_of(name)
    s, probs, thetas = handle(gar, name, B)
    d7 = d7_of(name)
    rng = np.random.default_rng(5)
    d = rng.standard_normal((nth, B, nth))  # nrhs = nth: the whole Jacobian's worth of directions
    out = sol(torch, d7, B, nth)
    s.theta_tangent(torch.from_numpy(d).cuda(), out)
    zs = {k: rng.standard_normal(tuple(v.shape[:1]) + tuple(v.shape[1:])) for k, v in sol(torch, d7, B, 2).items()}
    tb = torch.empty((2, B, nth), dtype=torch.float64, device="cuda")
    s.theta_adjoint({k: torch.from_numpy(v).cuda() for k, v in zs.items()}, tb)
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in out.items()}
    tb = tb.cpu().numpy()
    s.close()
    sub = [probs[b] for b in idx]
    o = lq_cases.oracle_parametric(sub, mueq, thetas[idx])
    J = [tref.theta_jacobian(p, mueq) for p in sub]
    ren = lambda z: {dict(lam0="lbd0", lams="lbdas").get(k, k): v for k, v in z.items()}
    per = [(j, i) for j in range(nth) for i in range(len(idx))]
    fac = [{k: o[k][i] for k in FAC} for i in range(len(idx))]
    gk = hp.stack_solutions([ren({k: v[j, idx[i]] for k, v in got.items()}) for j, i in per])
    ref = hp.stack_solutions([tref.jacobian_apply(J[i], d[j, idx[i]]) for j, i in per])
    ora = hp.stack_solutions([tref.tangent(fac[i], d[j, idx[i]], nu, nc) for j, i in per])
    e_kernel, e_oracle = tref.errors(gk, ref, nu, nc, N), tref.errors(ora, ref, nu, nc, N)
    print("\n" + hp.table("theta_tangent %s batch %d instances %s" % (name, B, idx), e_oracle, e_kernel))
    lq_cases.check_bar(e_kernel, e_oracle, "theta_tangent %s" % name)
    per = [(j, i) for j in range(2) for i in range(len(idx))]
    zr = ren(zs)
    pick = lambda j, i: {k: v[j, idx[i]] for k, v in zr.items()}
    ref = np.stack([tref.jacobian_transpose_apply(J[i], pick(j, i)) for j, i in per])
    ora = np.stack([tref.adjoint(fac[i], pick(j, i), nu, nc) for j, i in per])
    gk = np.stack([tb[j, idx[i]] for j, i in per])
    e_kernel, e_oracle = tref.theta_errors(gk, ref), tref.theta_errors(ora, ref)
    print(hp.table("theta_adjoint %s" % name, e_oracle, e_kernel))
    lq_cases.check_bar(e_kernel, e_oracle, "theta_adjoint %s" % name)


@pytest.mark.parametrize("name", ["c2_nth4", "c3_nth2"])
def test_transposition_and_affine_identity(env, name):
    gar, _, torch = env
    nx, nu, nc, nct, nc0, nth, N, mueq = CASES[name]
    B = 37
    s, probs, thetas = handle(gar, name, B)
    d7 = d7_of(name)
    rng = np.random.default_rng(8)
    d = torch.from_numpy(rng.standard_normal((1, B, nth))).cuda()
    jd = sol(torch, d7, B, 1)
    s.theta_tangent(d, jd)
    z = {k: torch.from_numpy(rng.standard_normal(tuple(v.shape))).cuda() for k, v in jd.items()}
    tb = torch.empty((1, B, nth), dtype=torch.float64, device="cuda")
    s.theta_adjoint(z, tb)
    terms = torch.stack([(z[k][0] * jd[k][0]).reshape(B, -1).sum(1) for k in KEYS if jd[k].numel()]).sum(0)
    scale = sum((z[k][0] * jd[k][0]).abs().reshape(B, -1).sum(1) for k in KEYS if jd[k].numel())
    rhs = (tb[0] * d[0]).sum(1)
    assert torch.all((terms - rhs).abs() <= 1e-12 * (scale + (tb[0] * d[0]).abs().sum(1)))
    # forward_theta(theta + d) - forward_theta(theta) = J d (device theta from a CUDA tensor)
    base = {k: s.get(w).copy() for k, w in zip(KEYS, (gar.OUT_XS, gar.OUT_US, gar.OUT_VS, gar.OUT_VST, gar.OUT_LBD0,
                                                      gar.OUT_LBDAS))}
    s.forward(theta=torch.from_numpy(thetas).cuda() + d[0])
    s.synchronize()
    for k, w in zip(KEYS, (gar.OUT_XS, gar.OUT_US, gar.OUT_VS, gar.OUT_VST, gar.OUT_LBD0, gar.OUT_LBDAS)):
        hi = s.get(w)
        if not hi.size:
            continue
        diff = hi - base[k]
        bound = 64 * hp.U * max(N, 1) * (np.abs(hi).max() + np.abs(base[k]).max())
        assert np.abs(diff - jd[k][0].cpu().numpy().reshape(diff.shape)).max() <= bound, k
    s.close()


def test_bit_invariance_across_nrhs_and_position(env):
    gar, _, torch = env
    name = "c3_nth2"
    nth = CASES[name][5]
    B = 11
    s, _, _ = handle(gar, name, B)
    d7 = d7_of(name)
    rng = np.random.default_rng(3)
    n = 40  # past one chunk of 32
    d = torch.from_numpy(rng.standard_normal((n, B, nth))).cuda()
    z = {k: torch.from_numpy(rng.standard_normal(tuple(v.shape))).cuda() for k, v in sol(torch, d7, B, n).items()}
    full = sol(torch, d7, B, n)
    s.theta_tangent(d, full)
    tbf = torch.empty((n, B, nth), dtype=torch.float64, device="cuda")
    s.theta_adjoint(z, tbf)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(1)).cuda()
    for sel in (perm, torch.tensor([35], device="cuda"), torch.tensor([2, 33, 7], device="cuda")):
        m = len(sel)
        part = sol(torch, d7, B, m)
        s.theta_tangent(d[sel].contiguous(), part)
        tb = torch.empty((m, B, nth), dtype=torch.float64, device="cuda")
        s.theta_adjoint({k: v[sel].contiguous() for k, v in z.items()}, tb)
        for k in KEYS:
            assert torch.equal(part[k], full[k][sel]), k
        assert torch.equal(tb, tbf[sel])
    s.close()


def snapshot(gar, s):
    outs = [s.get(w).copy() for w in range(20)]
    return outs, s.status().copy(), [p.copy() for p in s.pivot_stats()], s.factor_epoch()


def test_handle_unchanged(env):
    gar, _, torch = env
    name = "c3_nth2"
    B = 9
    s, _, _ = handle(gar, name, B)
    d7 = d7_of(name)
    nth = d7[5]
    before = snapshot(gar, s)
    out = sol(torch, d7, B, 3)
    s.theta_tangent(torch.ones((3, B, nth), dtype=torch.float64, device="cuda"), out)
    tb = torch.empty((3, B, nth), dtype=torch.float64, device="cuda")
    s.theta_adjoint({k: torch.ones_like(v) for k, v in out.items()}, tb)
    torch.cuda.synchronize()
    after = snapshot(gar, s)
    for a, b in zip(before[0], after[0]):
        assert np.array_equal(a, b, equal_nan=True)
    assert np.array_equal(before[1], after[1])
    assert all(np.array_equal(a, b) for a, b in zip(before[2], after[2]))
    assert before[3] == after[3]
    s.close()


def _tan(gar, s, nrhs, dtheta, out):
    ot = gar._fill(gar.LsIterate(), gar._LS_KEYS, out)
    p = None if dtheta is None else C.c_void_p(dtheta if isinstance(dtheta, int) else dtheta.data_ptr())
    return gar.lib().ab2_gar_theta_tangent(s.h, int(nrhs), p, C.byref(ot), None)


def _adj(gar, s, nrhs, cot, tb):
    ct = gar._fill(gar.LsIterate(), gar._LS_KEYS, cot)
    p = None if tb is None else C.c_void_p(tb if isinstance(tb, int) else tb.data_ptr())
    return gar.lib().ab2_gar_theta_adjoint(s.h, int(nrhs), C.byref(ct), p, None)


def test_return_codes(env):
    gar, _, torch = env
    name = "c3_nth2"
    nx, nu, nc, nct, nc0, nth, N, mueq = CASES[name]
    B = 5
    d7 = d7_of(name)
    out = sol(torch, d7, B, 2)
    dth = torch.zeros((2, B, nth), dtype=torch.float64, device="cuda")
    tb = torch.zeros((2, B, nth), dtype=torch.float64, device="cuda")
    cot = {k: torch.zeros_like(v) for k, v in out.items()}
    for kw in (dict(), dict(dense=True), dict(legs=2)):  # no parameters, dense, parallel
        u = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
        assert _tan(gar, u, 2, dth, out) == UNSUPPORTED, kw
        assert _adj(gar, u, 2, cot, tb) == UNSUPPORTED, kw
        u.close()
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, nth=nth)
    assert _tan(gar, s, 2, dth, out) == STATE and _adj(gar, s, 2, cot, tb) == STATE  # no problem
    s.set_problem(*gar.pack_problems(problems(name, B)))
    assert _tan(gar, s, 2, dth, out) == STATE and _adj(gar, s, 2, cot, tb) == STATE  # no backward since set_problem
    s.backward(mueq)
    s.synchronize()
    n0 = s.launch_count()
    assert _tan(gar, s, -1, dth, out) == INVALID and _adj(gar, s, -1, cot, tb) == INVALID
    assert _tan(gar, s, 2, None, out) == INVALID and _adj(gar, s, 2, cot, None) == INVALID
    for k in KEYS:
        if out[k].numel():
            bad = dict(out)
            bad[k] = None
            assert _tan(gar, s, 2, dth, bad) == INVALID, k
    # dtheta / cot overlapping out / theta_bar
    assert _tan(gar, s, 2, out["xs"], out) == INVALID
    assert _tan(gar, s, 2, out["lams"].reshape(-1)[3:], out) == INVALID
    assert _adj(gar, s, 2, dict(cot, us=tb), tb) == INVALID
    assert _adj(gar, s, 2, cot, cot["xs"].reshape(-1)[5:]) == INVALID
    # out / theta_bar overlapping an output of the handle
    for w in (gar.OUT_XS, gar.OUT_FTH, gar.OUT_KKT0FTH):
        assert _tan(gar, s, 1, dth, dict(out, us=s.device_ptr(w))) == INVALID, w
        assert _adj(gar, s, 1, cot, s.device_ptr(w)) == INVALID, w
    assert _tan(gar, s, 0, dth, out) == 0 and _adj(gar, s, 0, cot, tb) == 0
    assert s.launch_count() == n0  # nothing launched on an error or for nrhs = 0
    assert _tan(gar, s, 2, dth, out) == 0 and _adj(gar, s, 2, {}, tb) == 0
    assert s.launch_count() == n0 + 2
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# torch: autograd.lq_solve_theta
# ---------------------------------------------------------------------------------------------------------------------
def torch_case(env, name="c3_nth2", B=6):
    gar, ag, torch = env
    nx, nu, nc, nct, nc0, nth, N, mueq = CASES[name]
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, nth=nth)
    recs = [torch.from_numpy(np.ascontiguousarray(r)).cuda() for r in gar.pack_problems(problems(name, B))]
    theta = torch.from_numpy(np.random.default_rng(4).standard_normal((B, nth))).cuda()
    return s, recs, theta, mueq


def test_gradcheck(env):
    _, ag, torch = env
    s, recs, theta, mu = torch_case(env, B=2)
    f = lambda th: ag.lq_solve_theta(s, *recs, mu, th)
    assert torch.autograd.gradcheck(f, (theta.clone().requires_grad_(),), eps=1e-6, atol=1e-7, rtol=1e-6)
    assert torch.autograd.gradcheck(f, (theta.clone().requires_grad_(),), eps=1e-6, atol=1e-7, rtol=1e-6,
                                    check_forward_ad=True, check_backward_ad=False, check_undefined_grad=False)
    s.close()


def test_jacfwd_equals_jacrev_in_one_call_each(env):
    _, ag, torch = env
    s, recs, theta, mu = torch_case(env)
    f = lambda th: torch.cat([o.reshape(-1) for o in ag.lq_solve_theta(s, *recs, mu, th)])
    f(theta)
    n0 = s.launch_count()
    jr = torch.func.jacrev(f)(theta)
    n1 = s.launch_count()
    jf = torch.func.jacfwd(f)(theta)
    n2 = s.launch_count()
    sweep = n0  # the launches of one forward (set_problem has none; backward and forward_theta one each or more)
    assert n1 - n0 - sweep == 1 and n2 - n1 - sweep == 1, (n0, n1, n2)
    assert torch.allclose(jr, jf, rtol=1e-12, atol=1e-12 * jr.abs().max())
    s.close()


def test_hessian_of_a_quadratic_loss(env):
    _, ag, torch = env
    s, recs, theta, mu = torch_case(env, B=3)
    outs = ag.lq_solve_theta(s, *recs, mu, theta)
    w = [torch.rand_like(o) for o in outs]
    loss = lambda th: sum((wi * o * o).sum() for wi, o in zip(w, ag.lq_solve_theta(s, *recs, mu, th))) / 2
    H = torch.func.hessian(loss)(theta)
    f = lambda th: torch.cat([o.reshape(-1) for o in ag.lq_solve_theta(s, *recs, mu, th)])
    J = torch.func.jacfwd(f)(theta).reshape(-1, theta.numel())
    W = torch.cat([x.reshape(-1) for x in w])
    want = (J.T * W) @ J
    assert torch.allclose(H.reshape(want.shape), want, rtol=1e-10, atol=1e-10 * want.abs().max())
    s.close()


def test_refused_inputs(env):
    gar, ag, torch = env
    s, recs, theta, mu = torch_case(env)
    with pytest.raises(ValueError):
        ag.lq_solve_theta(s, *recs, mu, theta[:, :1].contiguous())
    with pytest.raises(ValueError):
        ag.lq_solve_theta(s, *recs, mu, theta.float())
    with pytest.raises(ValueError):
        ag.lq_solve_theta(s, *recs, mu, theta.cpu())
    for i in range(4):
        r = list(recs)
        r[i] = r[i].clone().requires_grad_()
        with pytest.raises(ValueError):
            ag.lq_solve_theta(s, *r, mu, theta)
    nx, nu, nc, nct, nc0, nth, N, _ = CASES["c3_nth2"]
    plain = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, theta.shape[0])
    with pytest.raises(ValueError):
        ag.lq_solve_theta(plain, *recs, mu, theta)
    plain.close()
    with pytest.raises(NotImplementedError):
        torch.func.vmap(lambda th: ag.lq_solve_theta(s, *recs, mu, th)[0])(torch.stack([theta, theta]))
    s.close()


def test_backward_after_another_call_refactors(env):
    _, ag, torch = env
    s, recs, theta, mu = torch_case(env)
    th = theta.clone().requires_grad_()
    xs = ag.lq_solve_theta(s, *recs, mu, th)[0]
    g0 = torch.autograd.grad(xs.square().sum(), th, retain_graph=True)[0]
    other = [r.clone() for r in recs]
    other[0].mul_(1.5)
    ag.lq_solve_theta(s, *other, mu, theta)  # refactors the handle on other data
    g1 = torch.autograd.grad(xs.square().sum(), th)[0]
    assert torch.equal(g0, g1)
    s.close()
