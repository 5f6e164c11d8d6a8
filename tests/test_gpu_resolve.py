"""Re-solving the last backward's LQ matrices for new vectors on the GPU (ab2_gar_resolve, gar.h;
aligator_b200.autograd.lq_resolve): parity with the oracle's solve of the problem with its vectors replaced, for every
non-dense handle kind of the adjoint tests; consistency with the sweep, the adjoint and the tangent; bit-exact
independence of nrhs; the handle's outputs untouched; state handling and errors; the per-instance-mu twin; full-size
configurations; and the torch entry point under autograd and torch.func."""
import ctypes as C

import numpy as np
import pytest

import gen
import lq_adjoint_ref as aref
import lq_gpu
import lq_resolve_ref as ref
from oracle import gar_oracle as orc
from lq_cases import BAR_CASES, bar_case, bar_violations
from lq_gpu import MUS, SERIAL

pytestmark = pytest.mark.gpu
TOL = 1e-10


@pytest.fixture(scope="module")
def env():
    return lq_gpu.gpu_env()


def _dev_rhs(env, h):
    _, _, torch = env
    return {k: torch.tensor(np.ascontiguousarray(v), device="cuda") for k, v in h.items()}


def _out(env, d6, B, nrhs):
    _, _, torch = env
    return {k: torch.full((nrhs,) + s, float("nan"), dtype=torch.float64, device="cuda")
            for k, s in zip(ref.SOL, ref.rhs_shapes(d6, B).values())}


def _oracle_replaced(recs, hj, d6, B, mu):
    nx, nu, nc, nct, nc0, N = d6
    bo = orc.BatchedOracle(nx, nu, nc, nct, nc0, N, B, *[np.ascontiguousarray(a) for a in
                                                         ref.replaced_records(*recs, hj, d6)])
    bo.sweep(mu)
    return aref.oracle_dict(bo.get())


def _close(z, want, tol, what, tol_vsT=None):
    for k in ref.SOL:
        t = tol_vsT if k == "vsT" and tol_vsT is not None else tol
        assert gen.rel_fro(z[k], want[k]) <= t, (what, k, gen.rel_fro(z[k], want[k]))


@pytest.mark.parametrize("mu", MUS)
@pytest.mark.parametrize("name,kw,dims", SERIAL, ids=[h[0] for h in SERIAL])
def test_parity_with_oracle(env, name, kw, dims, mu):
    nx, nu, nc, nct, nc0, N, B = dims
    d6 = dims[:6]
    s, recs = lq_gpu.setup(env, kw, dims, 3, mu)
    before = lq_gpu.outputs(env[0], s)
    h = ref.random_rhs(np.random.default_rng(4), d6, B, 3)
    out = _out(env, d6, B, 3)
    s.resolve(_dev_rhs(env, h), out, mu)
    z = lq_gpu.to_np(out)
    # v_N = (d_N + C_N x_N) / mu: x_N's rounding error reaches the terminal multipliers amplified by 1 / mu
    for j in range(3):
        _close({k: v[j] for k, v in z.items()}, _oracle_replaced(recs, {k: v[j] for k, v in h.items()}, d6, B, mu),
               TOL, (name, mu, j), tol_vsT=max(TOL, 1e-13 / mu))
    after = lq_gpu.outputs(env[0], s)
    for k, a in before.items():  # every handle output is bit-equal before and after
        assert np.array_equal(a, after[k], equal_nan=True), (name, k)
    s.close()


@pytest.mark.parametrize("name,kw,dims", [SERIAL[i] for i in (0, 8, 16, 17)],
                         ids=[SERIAL[i][0] for i in (0, 8, 16, 17)])
def test_consistency_with_sweep_adjoint_tangent(env, name, kw, dims):
    gar, _, torch = env
    nx, nu, nc, nct, nc0, N, B = dims
    d6 = dims[:6]
    mu = 1e-2
    s, recs = lq_gpu.setup(env, kw, dims, 5, mu)
    primal = {k: torch.tensor(s.get(w), device="cuda") for k, w in zip(
        aref.KEYS, (gar.OUT_XS, gar.OUT_US, gar.OUT_VS, gar.OUT_VST, gar.OUT_LBD0, gar.OUT_LBDAS))}
    stage, term, G0, g0 = recs
    so, _ = aref.stage_offsets(nx, nu, nc)
    to, _ = aref.term_offsets(nx, nct)
    st = stage.reshape(B, N, -1)
    vec = lambda n: st[..., so[n][0]:so[n][1]]
    own = dict(q=np.concatenate([vec("q"), term[:, None, to["q"][0]:to["q"][1]]], axis=1), r=vec("r"), d=vec("d"),
               dN=term[:, to["d"][0]:to["d"][1]], g0=g0, f=vec("f"))
    out = _out(env, d6, B, 1)
    s.resolve(_dev_rhs(env, {k: v[None] for k, v in own.items()}), out, mu)
    _close({k: v[0] for k, v in lq_gpu.to_np(out).items()}, {k: v.cpu().numpy() for k, v in primal.items()}, 1e-12, "primal")
    # -zbar gives the adjoint's trajectory
    rng = np.random.default_rng(6)
    zbar = {k: torch.tensor(rng.standard_normal(tuple(v.shape)), device="cuda") for k, v in primal.items()}
    grad = {k: torch.empty(sh, dtype=torch.float64, device="cuda") for k, sh in
            dict(stage=(B, N, s.srec), term=(B, s.trec), G0=(B, nc0 * nx), g0=(B, nc0)).items()}
    hz = dict(q=-zbar["xs"], r=-zbar["us"], d=-zbar["vs"], dN=-zbar["vsT"], g0=-zbar["lam0"], f=-zbar["lams"])
    out = _out(env, d6, B, 1)
    s.resolve({k: v[None].contiguous() for k, v in hz.items()}, out, mu)
    s.adjoint(primal, zbar, grad, mu)
    w = {k: s.get(wh) for k, wh in zip(ref.SOL, (gar.OUT_XS, gar.OUT_US, gar.OUT_VS, gar.OUT_VST, gar.OUT_LBD0,
                                                gar.OUT_LBDAS))}
    _close({k: v[0] for k, v in lq_gpu.to_np(out).items()}, w, TOL, "adjoint")
    # rho gives the tangent's trajectory (the handle is refactored by the adjoint: same matrices)
    import lq_tangent_ref as tref
    dot = dict(stage=rng.standard_normal((B, N, s.srec)), term=rng.standard_normal((B, s.trec)),
               G0=rng.standard_normal((B, nc0 * nx)), g0=rng.standard_normal((B, nc0)))
    pn = {k: v.cpu().numpy() for k, v in primal.items()}
    rho = tref.rho({k: v.reshape(v.shape[0], -1) if k != "stage" else v for k, v in dot.items()}, pn, d6)
    hr = dict(q=rho["xs"], r=rho["us"], d=rho["vs"], dN=rho["vsT"], g0=rho["lam0"], f=rho["lams"])
    out = _out(env, d6, B, 1)
    s.resolve(_dev_rhs(env, {k: v[None] for k, v in hr.items()}), out, mu)
    s.tangent(primal, _dev_rhs(env, dot), mu)
    zd = {k: s.get(wh) for k, wh in zip(ref.SOL, (gar.OUT_XS, gar.OUT_US, gar.OUT_VS, gar.OUT_VST, gar.OUT_LBD0,
                                                 gar.OUT_LBDAS))}
    _close({k: v[0] for k, v in lq_gpu.to_np(out).items()}, zd, TOL, "tangent")
    s.close()


@pytest.mark.parametrize("name,kw,dims", [SERIAL[i] for i in (0, 7, 16)], ids=[SERIAL[i][0] for i in (0, 7, 16)])
def test_bit_equal_across_nrhs_and_v_twin(env, name, kw, dims):
    gar, _, torch = env
    nx, nu, nc, nct, nc0, N, B = dims
    d6 = dims[:6]
    mu = 1e-2
    s, _ = lq_gpu.setup(env, kw, dims, 7, mu)
    for nrhs in (3, 32):
        h = _dev_rhs(env, ref.random_rhs(np.random.default_rng(nrhs), d6, B, nrhs))
        out = _out(env, d6, B, nrhs)
        s.resolve(h, out, mu)
        for j in (0, nrhs // 2, nrhs - 1):
            one = _out(env, d6, B, 1)
            s.resolve({k: v[j:j + 1].contiguous() for k, v in h.items()}, one, mu)
            for k in ref.SOL:
                assert torch.equal(one[k][0], out[k][j]), (name, nrhs, j, k)
    outv = _out(env, d6, B, 3)
    s.resolve({k: v[:3].contiguous() for k, v in h.items()}, outv, np.full(B, mu))
    outd = _out(env, d6, B, 3)
    s.resolve({k: v[:3].contiguous() for k, v in h.items()}, outd, torch.full((B,), mu, dtype=torch.float64,
                                                                              device="cuda"))
    for k in ref.SOL:
        assert torch.equal(outv[k], out[k][:3]) and torch.equal(outd[k], out[k][:3]), (name, k)
    # NULL fields are zero
    part = {k: (v[:2].contiguous() if k in ("q", "g0") else None) for k, v in h.items()}
    a, b = _out(env, d6, B, 2), _out(env, d6, B, 2)
    s.resolve(part, a, mu)
    s.resolve({k: (v if v is not None else torch.zeros_like(h[k][:2])) for k, v in part.items()}, b, mu)
    for k in ref.SOL:
        assert torch.equal(a[k], b[k]), k
    s.close()


def _rc(gar, s, mu, nrhs, rhs, out):
    rh = gar._fill(gar.LqRhs(), gar._RHS_KEYS, rhs)
    ot = gar._fill(gar.LsIterate(), gar._LS_KEYS, out)
    return gar.lib().ab2_gar_resolve(s.h, C.c_double(mu), int(nrhs), C.byref(rh), C.byref(ot), None)


def test_state_and_errors(env):
    gar, _, torch = env
    dims = (4, 2, 2, 2, 4, 6, 9)
    nx, nu, nc, nct, nc0, N, B = dims
    d6 = dims[:6]
    mu = 1e-2
    probs = gen.generate_batch(1, B, N, nx, nu, nc, nct)
    recs = gar.pack_problems(probs)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    out = _out(env, d6, B, 2)
    assert _rc(gar, s, mu, 2, {}, out) == 4  # no problem
    s.set_problem(*recs)
    assert _rc(gar, s, mu, 2, {}, out) == 4  # no backward since set_problem
    e0 = s.factor_epoch()
    s.sweep(mu)
    assert s.factor_epoch() > e0
    s.synchronize()
    n0 = s.launch_count()
    assert _rc(gar, s, mu, -1, {}, out) == 1
    assert _rc(gar, s, 0.0, 2, {}, out) == 1
    for k in ref.SOL:
        bad = dict(out)
        bad[k] = None
        assert _rc(gar, s, mu, 2, {}, bad) == 1, k
    assert _rc(gar, s, mu, 0, {}, out) == 0
    # an rhs array that overlaps an out array (an in-place q -> xs re-solve) is refused
    assert _rc(gar, s, mu, 2, dict(q=out["xs"]), out) == 1
    assert _rc(gar, s, mu, 2, dict(d=out["vs"][1:]), out) == 1
    assert _rc(gar, s, mu, 2, dict(f=out["xs"].reshape(-1)[nx:]), out) == 1
    assert s.launch_count() == n0  # nothing launched on an error or for nrhs = 0
    assert _rc(gar, s, mu, 2, {}, out) == 0
    assert s.launch_count() == n0 + 1
    # cycle_append, then a backward
    new_last = np.ascontiguousarray(gen.stage_record(gen.generate_batch(9, 1, 1, nx, nu, nc, nct)[0].stages[0]))
    _, srec = aref.stage_offsets(nx, nu, nc)
    nl = np.zeros((B, srec))
    nl[:, :new_last.size] = new_last
    s.cycle_append(nl)
    assert _rc(gar, s, mu, 2, {}, out) == 4
    s.sweep(mu)
    stage = s.get_problem(0).reshape(B, N, -1)
    term, G0, g0 = [s.get_problem(w).reshape(B, -1) for w in (1, 2, 3)]
    h = ref.random_rhs(np.random.default_rng(2), d6, B, 2)
    s.resolve(_dev_rhs(env, h), out, mu)
    z = lq_gpu.to_np(out)
    for j in range(2):
        _close({k: v[j] for k, v in z.items()},
               _oracle_replaced((stage, term, G0, g0), {k: v[j] for k, v in h.items()}, d6, B, mu), TOL, j)
    s.close()
    for kw in (dict(dense=True), dict(legs=2), dict(nth=2)):
        u = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
        assert _rc(gar, u, mu, 2, {}, out) == 2, kw
        u.close()


@pytest.mark.parametrize("dims", [(12, 6, 0, 0, 12, 100, 4096), (4, 2, 2, 2, 4, 100, 16384),
                                  (14, 7, 0, 0, 14, 200, 2048), (57, 28, 0, 0, 57, 150, 160)],
                         ids=["C2", "C3", "C4", "C5"])
def test_full_size(env, dims):
    gar, _, torch = env
    nx, nu, nc, nct, nc0, N, B = dims
    d6 = dims[:6]
    mu = 1e-2
    rng = np.random.default_rng(1)
    nrhs = 4
    s, recs = lq_gpu.setup(env, {}, dims, 2, mu)
    h = ref.random_rhs(rng, d6, B, nrhs)
    out = _out(env, d6, B, nrhs)
    s.resolve(_dev_rhs(env, h), out, mu)
    idx = np.r_[0:3, B // 2 - 2:B // 2 + 2, B - 5:B]  # first wave, a wave boundary, the ragged tail
    z = lq_gpu.to_np(out)
    st = recs[0].reshape(B, N, -1)
    sub = [np.ascontiguousarray(a[idx]) for a in (st, recs[1], recs[2].reshape(B, -1), recs[3].reshape(B, -1))]
    for j in (0, nrhs - 1):
        want = _oracle_replaced(sub, {k: v[j][idx] for k, v in h.items()}, d6, len(idx), mu)
        _close({k: v[j][idx] for k, v in z.items()}, want, TOL, j)
    s.close()


@pytest.mark.parametrize("name", list(BAR_CASES))
def test_device_meets_the_conditioning_bar(env, name):
    """Every trajectory family within max(16 e_oracle, 64 u) of the extended-precision solve of each replaced problem
    (DESIGN §5), on the device's own factorisation."""
    gar, _, _ = env
    probs, recs, case, mu, h = bar_case(name)
    nx, nu, nc, nct, nc0, N = case
    B = len(probs)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    s.set_problem(*[np.ascontiguousarray(a) for a in recs])
    s.sweep(mu)
    out = _out(env, case, B, 2)
    s.resolve(_dev_rhs(env, h), out, mu)
    z = lq_gpu.to_np(out)
    for j in range(2):
        bad, tab = bar_violations(probs, recs, case, mu, {k: v[j] for k, v in h.items()}, {k: v[j] for k, v in z.items()})
        assert not bad, "%s rhs %d\n%s" % (name, j, tab)
    s.close()


def test_torch_entry_point(env):
    gar, ag, torch = env
    dims = (4, 2, 2, 2, 4, 3, 2)
    nx, nu, nc, nct, nc0, N, B = dims
    d6 = dims[:6]
    mu = 1e-2
    s, recs = lq_gpu.setup(env, {}, dims, 9, mu)
    h = _dev_rhs(env, ref.random_rhs(np.random.default_rng(10), d6, B, 3))
    out = _out(env, d6, B, 3)
    s.resolve(h, out, mu)
    z = ag.lq_resolve(s, mu, **h)
    for k, zz in zip(ref.SOL, z):
        assert torch.equal(zz, out[k]), k
    # broadcast: unbatched fields are shared by every right-hand side
    z2 = ag.lq_resolve(s, mu, q=h["q"], g0=h["g0"][0])
    out2 = _out(env, d6, B, 3)
    s.resolve(dict(q=h["q"], g0=h["g0"][0:1].expand(3, -1, -1).contiguous()), out2, mu)
    for k, zz in zip(ref.SOL, z2):
        assert torch.equal(zz, out2[k]), k
    # gradcheck in both modes with respect to the vectors
    leaves = [h[k][0].clone().requires_grad_(True) for k in ("q", "r", "d", "dN", "g0", "f")]
    fn = lambda *a: ag.lq_resolve(s, mu, *a)
    assert torch.autograd.gradcheck(fn, leaves, check_forward_ad=True, check_backward_ad=True)
    # jacrev and jacfwd of xs with respect to g0 agree, and equal the columns of -K^-1 from the dense solve
    g0 = h["g0"][0].clone()
    fx = lambda g: ag.lq_resolve(s, mu, g0=g)[0]
    Jr = torch.func.jacrev(fx)(g0)
    Jf = torch.func.jacfwd(fx)(g0)
    assert torch.allclose(Jr, Jf, rtol=1e-12, atol=1e-14)
    probs = gen.generate_batch(9, B, N, nx, nu, nc, nct)
    for b in range(B):
        Kd, _, offs = gen.lqr_dense_kkt(probs[b], mu)
        Kinv = -np.linalg.inv(Kd)
        for t in range(N + 1):
            cols = Kinv[offs[t]:offs[t] + nx, :nc0]  # x_t against g0 (the first nc0 unknowns / rows)
            got = Jr[b, t, :, b, :].cpu().numpy()
            assert gen.rel_fro(got, cols) <= 1e-10, (b, t)
            assert float(Jr[b, t, :, 1 - b, :].abs().max()) == 0.0
    # vmap equals a Python loop
    qs = h["q"]
    vm = torch.func.vmap(lambda q: ag.lq_resolve(s, mu, q=q)[0])(qs)
    loop = torch.stack([ag.lq_resolve(s, mu, q=qs[i])[0] for i in range(3)])
    assert torch.equal(vm, loop)
    # a refactor between forward and backward raises
    q = h["q"][0].clone().requires_grad_(True)
    xs = ag.lq_resolve(s, mu, q=q)[0]
    s.sweep(mu)
    with pytest.raises(RuntimeError, match="refactored"):
        xs.sum().backward()
    s.close()
