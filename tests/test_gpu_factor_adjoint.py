"""Gradients of the factorisation on the GPU (ab2_gar_factor_adjoint, gar.h; aligator_b200.autograd.lq_factor): the
device against the numpy restatement fed with the device's own FF / FB / VXX / VX, on the warp kernel (packed Vxx) and
the CTA kernel (full Vxx), with constraints, horizons 0 and 1, forced 2x2 pivots, cycle_append, per-instance mu and NULL
cotangent fields; full-size C2 and C3 batches and C5 instances; untouched handle state, determinism and errors; and the
torch entry point under gradcheck, a mixed lq_solve / lq_factor loss, jacrev and jvp."""
import numpy as np
import pytest

import gen
import lq_adjoint_ref as aref
import lq_factor_adjoint_ref as ref
import lq_gpu
from lq_cases import block_errors, device_cot

pytestmark = pytest.mark.gpu
TOL = 1e-10
FAMS = ref.COT


@pytest.fixture(scope="module")
def env():
    return lq_gpu.gpu_env()


def _check(got, want, d6, tol, what):
    errs = block_errors(got, want, d6)
    assert max(errs.values()) <= tol, (what, errs)
    assert not got["G0"].any() and not got["g0"].any(), what  # zero-filled
    assert np.isfinite(got["stage"]).all(), what  # the pad double is written too


def _restate(recs, fac, cot, d6, mu):
    return ref.factor_adjoint(recs[0], recs[1], fac["ff"], fac["fb"], fac["vxx"], fac["vx"], fac["fft"], fac["fbt"],
                              cot, d6, mu)


@pytest.mark.parametrize("name,kw,dims,mu", lq_gpu.FACTOR_HANDLES, ids=[c[0] for c in lq_gpu.FACTOR_HANDLES])
def test_matches_restatement(env, name, kw, dims, mu):
    gar, _, _ = env
    d6 = dims[:6]
    B = dims[6]
    probs = gen.generate_batch(41, B, dims[5], *dims[:3], dims[3])
    recs = lq_gpu.handle_records(gar, probs)
    s = gar.CudaRiccatiBatch(*dims, **kw)
    s.set_problem(*recs)
    s.backward(mu)
    cot = ref.random_cot(np.random.default_rng(2), d6, B)
    got = lq_gpu.device_factor_adjoint(env, s, cot, mu, d6)
    _check(got, _restate(recs, lq_gpu.factor(gar, s), cot, d6, mu), d6, max(TOL, 2.4e-16 / mu), name)
    # NULL fields are zero cotangents; FB alone
    for part in (dict(fb=cot["fb"]), dict(cot, vxx=None, fft=None), dict(vxx=cot["vxx"], vx=cot["vx"])):
        got = lq_gpu.device_factor_adjoint(env, s, part, mu, d6)
        _check(got, _restate(recs, lq_gpu.factor(gar, s), part, d6, mu), d6, max(TOL, 2.4e-16 / mu), (name, list(part)))
    s.close()


def test_forced_2x2_pivots_cycle_append_and_per_instance_mu(env):
    gar, _, torch = env
    dims = (4, 2, 2, 2, 4, 6, 6)
    nx, nu, nc, nct, nc0, N, B = dims
    d6 = dims[:6]
    probs = gen.generate_batch(42, B, N, nx, nu, nc, nct)
    gen.make_2x2_pivots(probs)
    recs = lq_gpu.handle_records(gar, probs)
    s = gar.CudaRiccatiBatch(*dims)
    s.set_problem(*recs)
    mu = np.array([1e-3, 1e-2, 1e-3, 1e-1, 1e-3, 1e-2])
    s.backward(mu)
    assert s.pivot_stats()[0].sum() > 0  # the 2x2 pivot path ran
    cot = ref.random_cot(np.random.default_rng(3), d6, B)
    _check(lq_gpu.device_factor_adjoint(env, s, cot, mu, d6), _restate(recs, lq_gpu.factor(gar, s), cot, d6, mu), d6, TOL, "2x2 _v")
    # cycle_append, then a backward: records are read through the ring head
    _, srec = aref.stage_offsets(nx, nu, nc)
    new = gen.generate_batch(43, B, 1, nx, nu, nc, nct)
    nl = np.stack([np.pad(gen.stage_record(p.stages[0]), (0, srec - gen.stage_record(p.stages[0]).size))
                   for p in new])
    s.cycle_append(np.ascontiguousarray(nl))
    with pytest.raises(gar.GarError, match="error 4"):
        lq_gpu.device_factor_adjoint(env, s, cot, 1e-3, d6)
    s.backward(1e-3)
    stage = s.get_problem(0).reshape(B, N, -1)
    term = s.get_problem(1).reshape(B, -1)
    _check(lq_gpu.device_factor_adjoint(env, s, cot, 1e-3, d6), _restate((stage, term), lq_gpu.factor(gar, s), cot, d6, 1e-3), d6, TOL, "cycle")
    s.close()


def test_state_untouched_deterministic_and_errors(env):
    gar, _, torch = env
    dims = (4, 2, 2, 2, 4, 5, 7)
    nx, nu, nc, nct, nc0, N, B = dims
    d6 = dims[:6]
    mu = 1e-3
    recs = lq_gpu.handle_records(gar, gen.generate_batch(44, B, N, nx, nu, nc, nct))
    s = gar.CudaRiccatiBatch(*dims)
    s.set_problem(*recs)
    cot = ref.random_cot(np.random.default_rng(4), d6, B)
    with pytest.raises(gar.GarError, match="error 4"):  # no backward since set_problem
        lq_gpu.device_factor_adjoint(env, s, cot, mu, d6)
    s.sweep(mu)
    before, e0 = lq_gpu.outputs(gar, s), s.factor_epoch()
    a1 = lq_gpu.device_factor_adjoint(env, s, cot, mu, d6)
    a2 = lq_gpu.device_factor_adjoint(env, s, cot, mu, d6)
    for k in a1:
        assert np.array_equal(a1[k], a2[k]), k  # two calls, identical bits
    after = lq_gpu.outputs(gar, s)
    for k, v in before.items():
        assert np.array_equal(v, after[k], equal_nan=True), k
    assert s.factor_epoch() == e0
    # errors: nothing is launched
    g = lq_gpu.grads(torch, s)
    dc = {k: lq_gpu.dev(torch, v) for k, v in device_cot(cot, d6, B).items()}
    n0 = s.launch_count()
    with pytest.raises(gar.GarError, match="error 1"):
        s.factor_adjoint(dc, g, 0.0)
    with pytest.raises(gar.GarError, match="error 1"):  # a cotangent inside the grad array
        s.factor_adjoint(dict(dc, ff=g["stage"].reshape(-1)[:B * N * (nu + nc + nx)]), g, mu)
    assert s.launch_count() == n0
    # after an adjoint or a tangent FF and VX hold that solve's vectors
    primal = {k: torch.tensor(np.ascontiguousarray(s.get(w)), device="cuda")
              for k, w in zip(aref.KEYS, (gar.OUT_XS, gar.OUT_US, gar.OUT_VS, gar.OUT_VST, gar.OUT_LBD0,
                                          gar.OUT_LBDAS))}
    s.adjoint(primal, dict(xs=torch.ones_like(primal["xs"])), {}, mu)
    with pytest.raises(gar.GarError, match="error 4"):
        s.factor_adjoint(dc, g, mu)
    s.backward(mu)
    s.factor_adjoint(dc, g, mu)
    s.tangent(primal, dict(stage=torch.ones((B, N, s.srec), dtype=torch.float64, device="cuda")), mu)
    with pytest.raises(gar.GarError, match="error 4"):
        s.factor_adjoint(dc, g, mu)
    s.close()
    for kw in (dict(dense=True), dict(legs=2), dict(nth=2)):
        u = gar.CudaRiccatiBatch(*dims, **kw)
        n0 = u.launch_count()
        with pytest.raises(gar.GarError, match="error 2"):
            u.factor_adjoint(dc, g, mu)
        assert u.launch_count() == n0, kw
        u.close()


@pytest.mark.parametrize("cfg", [("C2", 12, 6, 0, 0, 100, 4096, 1e-2), ("C3", 4, 2, 2, 2, 100, 16384, 1e-3),
                                 ("C5", 57, 28, 0, 0, 40, 200, 1e-2)], ids=["C2", "C3", "C5"])
def test_full_size(env, cfg):
    gar, _, torch = env
    import bench
    name, nx, nu, nc, nct, N, B, mu = cfg
    d6 = (nx, nu, nc, nct, nx, N)
    stage, term, G0, g0 = bench.synth_batch_torch(torch, B, N, nx, nu, "cuda:0", 77, nc, nct, "control")
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nx, N, B)
    s.set_problem(stage, term, G0, g0, memspace=gar.AB2_DEVICE)
    s.backward(mu)
    assert np.all(s.status() == 0)
    gen_t = torch.Generator(device="cuda").manual_seed(5)
    shapes = ref.cot_shapes(d6, B)
    cot = {k: torch.randn(v, dtype=torch.float64, device="cuda", generator=gen_t) for k, v in shapes.items()}
    dc = {k: (v.transpose(-1, -2).contiguous() if k == "vxx" else v) for k, v in cot.items()}
    g = lq_gpu.grads(torch, s)
    s.factor_adjoint(dc, g, mu)
    s.synchronize()
    # the first wave, a wave boundary and the ragged tail (C5: a few instances)
    blocks = [(0, 24), (B // 2 - 8, 16), (B - 24, 24)] if name != "C5" else [(0, 2), (B - 2, 2)]
    for b0, nb in blocks:
        sl = slice(b0, b0 + nb)
        fac = {}
        for k, w in zip(FAMS, (gar.OUT_FF, gar.OUT_FB, gar.OUT_VXX, gar.OUT_VX, gar.OUT_FFT, gar.OUT_FBT)):
            per = int(np.prod(s.out_shape(w)[1:]))
            buf = np.empty(max(nb * per, 1))
            if per:
                t1 = s.out_shape(w)[1] if w in (gar.OUT_FF, gar.OUT_FB, gar.OUT_VXX, gar.OUT_VX) else 1
                s.get_range_into(w, b0, nb, 0, t1, buf, gar.AB2_HOST)
            s.synchronize()
            a = buf[:nb * per].reshape((nb,) + s.out_shape(w)[1:])
            fac[k] = np.swapaxes(a, -1, -2) if w == gar.OUT_VXX else a
        recs = (stage[sl].cpu().numpy(), term[sl].cpu().numpy())
        want = _restate(recs, fac, {k: v[sl].cpu().numpy() for k, v in cot.items()}, d6, mu)
        got = {k: v[sl].cpu().numpy() for k, v in g.items()}
        _check(got, want, d6, TOL, (name, b0))
    s.close()


# ---- torch ----
def test_gradcheck_lq_factor(env):
    gar, ag, torch = env
    nx, nu, nc, nct, nc0, N, B = 4, 2, 2, 2, 4, 3, 2
    probs = gen.generate_batch(21, B, N, nx, nu, nc, nct)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    blocks, term, init = lq_gpu.block_inputs(torch, probs)
    names = list(blocks) + ["t" + n for n in term]
    leaves = list(blocks.values()) + list(term.values())
    sym = lambda P: 0.5 * (P + P.transpose(-1, -2))
    G0, g0 = [t.detach().contiguous() for t in init.values()]

    def f(*xs):
        a = dict(zip(names, xs))
        st = ag.stage_records(a["A"], a["B"], a["f"], sym(a["Q"]), a["S"], sym(a["R"]), a["q"], a["r"], a["C"], a["D"],
                              a["d"])
        tt = ag.term_records(sym(a["tQ"]), a["tq"], a["tC"], a["td"])
        return ag.lq_factor(s, st.contiguous(), tt.contiguous(), G0, g0, 1e-2)

    assert torch.autograd.gradcheck(f, tuple(leaves), eps=1e-6, atol=1e-6, rtol=1e-4)
    s.close()


def _torch_solution(fac, G0, g0, case):
    """The LQ solution from a torch factorisation (ref.torch_factor) and the initial condition, differentiably."""
    import torch
    nx, nu, nc, nct, nc0, N = case
    B = G0.shape[0]
    V0, v0 = fac["vxx"][:, 0], fac["vx"][:, 0]
    G = G0.reshape(B, nx, nc0).transpose(-1, -2)
    M = torch.cat([torch.cat([V0, G.transpose(-1, -2)], -1),
                   torch.cat([G, torch.zeros(B, nc0, nc0, dtype=torch.float64)], -1)], -2)
    s0 = -torch.linalg.solve(M, torch.cat([v0, g0], -1)[..., None])[..., 0]
    x = s0[:, :nx]
    xs, us, vs, ls = [x], [], [], []
    for t in range(N):
        F, f = fac["fb"][:, t], fac["ff"][:, t]
        y = f + (F @ x[..., None])[..., 0]
        us.append(y[:, :nu])
        vs.append(y[:, nu:nu + nc])
        x = y[:, nu + nc:]
        xs.append(x)
        ls.append(fac["vx"][:, t + 1] + (fac["vxx"][:, t + 1] @ x[..., None])[..., 0])
    vsT = fac["fft"] + (fac["fbt"] @ x[..., None])[..., 0]
    st = lambda a, w: torch.stack(a, 1) if a else torch.zeros(B, 0, w, dtype=torch.float64)
    return dict(xs=torch.stack(xs, 1), us=st(us, nu), vs=st(vs, nc), vsT=vsT, lam0=s0[:, nx:], lams=st(ls, nx))


def test_mixed_loss_jacrev_and_jvp(env):
    gar, ag, torch = env
    case = (4, 2, 2, 2, 4, 4)
    nx, nu, nc, nct, nc0, N = case
    B, mu = 2, 1e-2
    recs = lq_gpu.handle_records(gar, gen.general_initial_condition(gen.generate_batch(45, B, N, nx, nu, nc, nct), nc0, 45))
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    rng = np.random.default_rng(6)
    dev = [torch.tensor(np.ascontiguousarray(a), device="cuda", requires_grad=True) for a in recs]
    cs = {k: rng.standard_normal(v.shape) for k, v in zip(aref.KEYS, [np.zeros(sh) for sh in (
        (B, N + 1, nx), (B, N, nu), (B, N, nc), (B, nct), (B, nc0), (B, N, nx))])}
    cf = ref.random_cot(rng, case, B)
    # lq_factor first, then lq_solve: each backward re-sets the problem
    fo = ag.lq_factor(s, *dev, mu)
    so = ag.lq_solve(s, *dev, mu)
    loss = sum((o * torch.tensor(cf[k], device="cuda")).sum() for k, o in zip(FAMS, fo)) + \
        sum((o * torch.tensor(cs[k], device="cuda")).sum() for k, o in zip(aref.KEYS, so))
    gd = torch.autograd.grad(loss, dev)
    cpu = [torch.tensor(a, requires_grad=True) for a in recs]
    fac = ref.torch_factor(cpu[0], cpu[1], case, mu)
    sol = _torch_solution(fac, cpu[2], cpu[3], case)
    lc = sum((fac[k] * torch.tensor(cf[k])).sum() for k in FAMS) + \
        sum((sol[k] * torch.tensor(cs[k])).sum() for k in aref.KEYS)
    gc = torch.autograd.grad(lc, cpu)
    for name, a, b in zip(("stage", "term", "G0", "g0"), gd, gc):
        assert gen.rel_fro(a.cpu().numpy(), b.numpy()) <= 1e-9, name
    # jacrev of K_0 with respect to the stage records
    st0 = dev[0].detach()
    rest = [t.detach() for t in dev[1:]]
    K0 = lambda st: ag.lq_factor(s, st, *rest, mu)[1][:, 0, :nu, :]
    J = torch.func.jacrev(K0)(st0).cpu().numpy()
    Jc = torch.autograd.functional.jacobian(
        lambda st: ref.torch_factor(st, torch.tensor(recs[1]), case, mu)["fb"][:, 0, :nu, :], torch.tensor(recs[0]))
    # the oracle's gradient is the symmetric-argument one for Q and R: compare on a symmetric direction
    so_, _ = aref.stage_offsets(nx, nu, nc)
    d = rng.standard_normal(recs[0].shape)
    for key, k in (("Q", nx), ("R", nu)):
        blk = d[..., so_[key][0]:so_[key][1]].reshape(B, N, k, k)
        d[..., so_[key][0]:so_[key][1]] = (blk + np.swapaxes(blk, -1, -2)).reshape(B, N, k * k)
    lead = J.ndim - 3
    jd = np.tensordot(J, d, axes=3)
    jcd = np.tensordot(Jc.numpy(), d, axes=3)
    assert lead == 3 and gen.rel_fro(jd, jcd) <= 1e-9
    with pytest.raises(NotImplementedError, match="forward mode of the gains"):
        torch.func.jvp(K0, (st0,), (torch.ones_like(st0),))
    with pytest.raises(NotImplementedError):
        torch.func.vmap(lambda st: ag.lq_factor(s, st, *rest, mu)[0])(st0[None].expand(2, *st0.shape).contiguous())
    s.close()
