"""Forward mode of the factorisation on the GPU (ab2_gar_factor_tangent, gar.h; aligator_b200.autograd.lq_factor_fwd):
the device against the numpy restatement fed with the device's own FF / FB / VXX / VX, on the warp kernel (packed Vxx)
and the CTA kernel (full Vxx), with constraints, horizons 0 and 1, forced 2x2 pivots, cycle_append, per-instance mu,
NULL tangent fields and NULL out fields; duality with ab2_gar_factor_adjoint; full-size C2 and C3 batches and C5
instances; untouched handle state, determinism and errors; and the torch entry point under jvp, gradcheck and
jacfwd."""
import numpy as np
import pytest

import gen
import lq_adjoint_ref as aref
import lq_factor_adjoint_ref as adj
import lq_factor_tangent_ref as ref
import lq_gpu
from lq_cases import device_cot, family_errors, random_dot

pytestmark = pytest.mark.gpu
TOL = 1e-10
FAMS = adj.COT


@pytest.fixture(scope="module")
def env():
    return lq_gpu.gpu_env()


def _restate(recs, fac, dot, d6, mu):
    return ref.factor_tangent(recs[0], recs[1], fac["ff"], fac["fb"], fac["vxx"], fac["vx"], fac["fft"], fac["fbt"],
                              dot, d6, mu)


def _check(got, want, tol, what, fams=FAMS):
    errs = {k: e for k, e in family_errors(got, want).items() if k in fams}
    assert not errs or max(errs.values()) <= tol, (what, errs)
    assert np.array_equal(got["vxx"], np.swapaxes(got["vxx"], -1, -2)) or "vxx" not in fams, what


@pytest.mark.parametrize("name,kw,dims,mu", lq_gpu.FACTOR_HANDLES, ids=[c[0] for c in lq_gpu.FACTOR_HANDLES])
def test_matches_restatement(env, name, kw, dims, mu):
    gar, _, _ = env
    d6 = dims[:6]
    B = dims[6]
    probs = gen.generate_batch(61, B, dims[5], *dims[:3], dims[3])
    recs = lq_gpu.handle_records(gar, probs)
    s = gar.CudaRiccatiBatch(*dims, **kw)
    s.set_problem(*recs)
    s.backward(mu)
    dot = random_dot(np.random.default_rng(21), d6, B)
    tol = max(TOL, 2.4e-16 / mu)
    fac = lq_gpu.factor(gar, s)
    _check(lq_gpu.device_factor_tangent(env, s, dot, mu, d6), _restate(recs, fac, dot, d6, mu), tol, name)
    # NULL tangent fields are zero: stage only, term only
    for part in (dict(stage=dot["stage"]), dict(term=dot["term"])):
        _check(lq_gpu.device_factor_tangent(env, s, part, mu, d6), _restate(recs, fac, part, d6, mu), tol, (name, list(part)))
    # NULL out fields are not written
    got = lq_gpu.device_factor_tangent(env, s, dot, mu, d6, want=("fb", "vx"))
    _check(got, _restate(recs, fac, dot, d6, mu), tol, (name, "fb vx"), fams=("fb", "vx"))
    for k in ("ff", "vxx", "fft", "fbt"):
        assert np.isnan(got[k]).all(), (name, k)
    s.close()


def test_forced_2x2_pivots_cycle_append_and_per_instance_mu(env):
    gar, _, torch = env
    dims = (4, 2, 2, 2, 4, 6, 6)
    nx, nu, nc, nct, nc0, N, B = dims
    d6 = dims[:6]
    probs = gen.generate_batch(62, B, N, nx, nu, nc, nct)
    gen.make_2x2_pivots(probs)
    recs = lq_gpu.handle_records(gar, probs)
    s = gar.CudaRiccatiBatch(*dims)
    s.set_problem(*recs)
    mu = np.array([1e-3, 1e-2, 1e-3, 1e-1, 1e-3, 1e-2])
    s.backward(mu)
    assert s.pivot_stats()[0].sum() > 0  # the 2x2 pivot path ran
    dot = random_dot(np.random.default_rng(22), d6, B)
    _check(lq_gpu.device_factor_tangent(env, s, dot, mu, d6), _restate(recs, lq_gpu.factor(gar, s), dot, d6, mu), TOL, "2x2 _v")
    # cycle_append, then a backward: records are read through the ring head
    _, srec = aref.stage_offsets(nx, nu, nc)
    new = gen.generate_batch(63, B, 1, nx, nu, nc, nct)
    nl = np.stack([np.pad(gen.stage_record(p.stages[0]), (0, srec - gen.stage_record(p.stages[0]).size))
                   for p in new])
    s.cycle_append(np.ascontiguousarray(nl))
    with pytest.raises(gar.GarError, match="error 4"):
        lq_gpu.device_factor_tangent(env, s, dot, 1e-3, d6)
    s.backward(1e-3)
    stage = s.get_problem(0).reshape(B, N, -1)
    term = s.get_problem(1).reshape(B, -1)
    _check(lq_gpu.device_factor_tangent(env, s, dot, 1e-3, d6), _restate((stage, term), lq_gpu.factor(gar, s), dot, d6, 1e-3), TOL, "cycle")
    s.close()


def test_state_untouched_deterministic_and_errors(env):
    gar, _, torch = env
    dims = (4, 2, 2, 2, 4, 5, 7)
    nx, nu, nc, nct, nc0, N, B = dims
    d6 = dims[:6]
    mu = 1e-3
    recs = lq_gpu.handle_records(gar, gen.generate_batch(64, B, N, nx, nu, nc, nct))
    s = gar.CudaRiccatiBatch(*dims)
    s.set_problem(*recs)
    dot = random_dot(np.random.default_rng(23), d6, B)
    with pytest.raises(gar.GarError, match="error 4"):  # no backward since set_problem
        lq_gpu.device_factor_tangent(env, s, dot, mu, d6)
    s.sweep(mu)
    before, e0 = lq_gpu.outputs(gar, s), s.factor_epoch()
    a1 = lq_gpu.device_factor_tangent(env, s, dot, mu, d6)
    a2 = lq_gpu.device_factor_tangent(env, s, dot, mu, d6)
    for k in a1:
        assert np.array_equal(a1[k], a2[k]), k  # two calls, identical bits
    after = lq_gpu.outputs(gar, s)
    for k, v in before.items():
        assert np.array_equal(v, after[k], equal_nan=True), k
    assert s.factor_epoch() == e0
    # errors: nothing is launched
    o = lq_gpu.outs(torch, d6, B)
    dd = {k: lq_gpu.dev(torch, v) for k, v in dot.items()}
    n0 = s.launch_count()
    with pytest.raises(gar.GarError, match="error 1"):
        s.factor_tangent(dd, o, 0.0)
    with pytest.raises(gar.GarError, match="error 1"):  # an out array inside a dot array
        s.factor_tangent(dd, dict(o, vx=dd["stage"].reshape(-1)[:B * (N + 1) * nx]), mu)
    with pytest.raises(gar.GarError, match="error 1"):  # an out array inside an output of the handle
        s.factor_tangent(dd, dict(o, ff=s.device_ptr(gar.OUT_XS)), mu)
    assert s.launch_count() == n0
    # after an adjoint or a tangent FF and VX hold that solve's vectors
    primal = {k: torch.tensor(np.ascontiguousarray(s.get(w)), device="cuda")
              for k, w in zip(aref.KEYS, (gar.OUT_XS, gar.OUT_US, gar.OUT_VS, gar.OUT_VST, gar.OUT_LBD0,
                                          gar.OUT_LBDAS))}
    s.adjoint(primal, dict(xs=torch.ones_like(primal["xs"])), {}, mu)
    with pytest.raises(gar.GarError, match="error 4"):
        s.factor_tangent(dd, o, mu)
    s.backward(mu)
    s.factor_tangent(dd, o, mu)
    s.tangent(primal, dict(stage=torch.ones((B, N, s.srec), dtype=torch.float64, device="cuda")), mu)
    with pytest.raises(gar.GarError, match="error 4"):
        s.factor_tangent(dd, o, mu)
    s.close()
    for kw in (dict(dense=True), dict(legs=2), dict(nth=2)):
        u = gar.CudaRiccatiBatch(*dims, **kw)
        n0 = u.launch_count()
        with pytest.raises(gar.GarError, match="error 2"):
            u.factor_tangent(dd, o, mu)
        assert u.launch_count() == n0, kw
        u.close()


@pytest.mark.parametrize("name,kw,dims,mu", [lq_gpu.FACTOR_HANDLES[0], lq_gpu.FACTOR_HANDLES[1], lq_gpu.FACTOR_HANDLES[4], lq_gpu.FACTOR_HANDLES[7]],
                         ids=[lq_gpu.FACTOR_HANDLES[i][0] for i in (0, 1, 4, 7)])
def test_duality_with_factor_adjoint(env, name, kw, dims, mu):
    """<cbar, ydot> from factor_tangent = <factor_adjoint(cbar), pdot>, both on the device: within 1e-10 relative, or
    at small mu within the conditioning bar max(1e-10, 2.4e-16 / mu) of the two calls' own results (the pairings grow
    like 1/mu with terminal constraints)."""
    gar, _, torch = env
    d6 = dims[:6]
    B = dims[6]
    recs = lq_gpu.handle_records(gar, gen.generate_batch(65, B, dims[5], *dims[:3], dims[3]))
    s = gar.CudaRiccatiBatch(*dims, **kw)
    s.set_problem(*recs)
    s.backward(mu)
    rng = np.random.default_rng(24)
    for _ in range(2):
        dot = random_dot(rng, d6, B)
        cot = adj.random_cot(rng, d6, B)
        tan = lq_gpu.device_factor_tangent(env, s, dot, mu, d6)
        dc = {k: lq_gpu.dev(torch, v) for k, v in device_cot(cot, d6, B).items()}
        g = lq_gpu.grads(torch, s)
        s.factor_adjoint(dc, g, mu)
        s.synchronize()
        lhs = sum(float((tan[k] * cot[k]).sum()) for k in FAMS)
        rhs = float((g["stage"].cpu().numpy() * dot["stage"]).sum() + (g["term"].cpu().numpy() * dot["term"]).sum())
        assert abs(lhs - rhs) <= max(1e-10, 2.4e-16 / mu) * max(abs(lhs), 1.0), (name, lhs, rhs)
    s.close()


@pytest.mark.parametrize("cfg", [("C2", 12, 6, 0, 0, 100, 4096, 1e-2), ("C3", 4, 2, 2, 2, 100, 16384, 1e-3),
                                 ("C5", 57, 28, 0, 0, 40, 200, 1e-2)], ids=["C2", "C3", "C5"])
def test_full_size(env, cfg):
    gar, _, torch = env
    import bench
    name, nx, nu, nc, nct, N, B, mu = cfg
    d6 = (nx, nu, nc, nct, nx, N)
    stage, term, G0, g0 = bench.synth_batch_torch(torch, B, N, nx, nu, "cuda:0", 78, nc, nct, "control")
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nx, N, B)
    s.set_problem(stage, term, G0, g0, memspace=gar.AB2_DEVICE)
    s.backward(mu)
    assert np.all(s.status() == 0)
    gen_t = torch.Generator(device="cuda").manual_seed(6)
    dot = dict(stage=torch.randn(stage.shape, dtype=torch.float64, device="cuda", generator=gen_t),
               term=torch.randn(term.shape, dtype=torch.float64, device="cuda", generator=gen_t))
    o = lq_gpu.outs(torch, d6, B)
    s.factor_tangent(dot, o, mu)
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
        want = _restate(recs, fac, {k: v[sl].cpu().numpy() for k, v in dot.items()}, d6, mu)
        got = {k: (np.swapaxes(v[sl].cpu().numpy(), -1, -2) if k == "vxx" else v[sl].cpu().numpy())
               for k, v in o.items()}
        _check(got, want, TOL, (name, b0))
    s.close()


# ---- torch ----
def _torch_case(env, seed, case=(4, 2, 2, 2, 4, 4), B=2):
    gar, ag, torch = env
    nx, nu, nc, nct, nc0, N = case
    recs = lq_gpu.handle_records(gar, gen.general_initial_condition(gen.generate_batch(seed, B, N, nx, nu, nc, nct), nc0, seed))
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    dev = [torch.tensor(np.ascontiguousarray(a), device="cuda") for a in recs]
    return s, recs, dev


def test_lq_factor_fwd_outputs_and_jvp(env):
    gar, ag, torch = env
    case = (4, 2, 2, 2, 4, 4)
    mu = 1e-2
    s, recs, dev = _torch_case(env, 66, case)
    a = ag.lq_factor(s, *dev, mu)
    b = ag.lq_factor_fwd(s, *dev, mu)
    for k, x, y in zip(FAMS, a, b):
        assert torch.equal(x, y), k  # bit for bit
    dot = random_dot(np.random.default_rng(25), case, 2)
    dd = [torch.tensor(dot["stage"], device="cuda"), torch.tensor(dot["term"], device="cuda")]
    rest = dev[2:]
    prim, tan = torch.func.jvp(lambda st, tt: ag.lq_factor_fwd(s, st, tt, *rest, mu), tuple(dev[:2]), tuple(dd))
    for k, x, y in zip(FAMS, prim, a):
        assert torch.equal(x, y), k
    fac = {k: v.cpu().numpy() for k, v in zip(FAMS, a)}
    want = _restate(recs, fac, dot, case, mu)
    errs = family_errors({k: v.cpu().numpy() for k, v in zip(FAMS, tan)}, want)
    assert max(errs.values()) <= TOL, errs
    # forward_ad gives the same tangents
    import torch.autograd.forward_ad as fwAD
    with fwAD.dual_level():
        st = fwAD.make_dual(dev[0], dd[0])
        tt = fwAD.make_dual(dev[1], dd[1])
        out = ag.lq_factor_fwd(s, st, tt, *rest, mu)
        for k, o, t in zip(FAMS, out, tan):
            assert torch.equal(fwAD.unpack_dual(o).tangent, t), k
    s.close()


def test_gradcheck_forward_mode(env):
    gar, ag, torch = env
    nx, nu, nc, nct, nc0, N, B = 4, 2, 2, 2, 4, 3, 2
    probs = gen.generate_batch(67, B, N, nx, nu, nc, nct)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    blocks, term, init = lq_gpu.block_inputs(torch, probs)
    names = list(blocks) + ["t" + n for n in term]
    leaves = list(blocks.values()) + list(term.values())
    sym = lambda P: 0.5 * (P + P.transpose(-1, -2))  # the sweep reads Q and R as symmetric
    G0, g0 = [t.detach().contiguous() for t in init.values()]

    def f(*xs):
        a = dict(zip(names, xs))
        st = ag.stage_records(a["A"], a["B"], a["f"], sym(a["Q"]), a["S"], sym(a["R"]), a["q"], a["r"], a["C"], a["D"],
                              a["d"])
        tt = ag.term_records(sym(a["tQ"]), a["tq"], a["tC"], a["td"])
        return ag.lq_factor_fwd(s, st.contiguous(), tt.contiguous(), G0, g0, 1e-2)

    assert torch.autograd.gradcheck(f, tuple(leaves), eps=1e-6, atol=1e-6, rtol=1e-4, check_forward_ad=True,
                                    check_backward_ad=False, check_undefined_grad=False)
    s.close()


def test_jacfwd_matches_jacrev_and_refusals(env):
    gar, ag, torch = env
    case = (4, 2, 2, 2, 4, 4)
    nx, nu, nc, nct, nc0, N = case
    mu = 1e-2
    s, recs, dev = _torch_case(env, 68, case)
    rest = dev[1:]
    so, _ = aref.stage_offsets(nx, nu, nc)
    # a few stage entries: A_0[1, 2], B_1[0, 1], f_2[3] and Q_0[2, 1] of instance 0, as a parameter vector
    idx = [(0, 0, 1 + 2 * nx), (0, 1, so["B"][0] + 0 + 1 * nx), (0, 2, so["f"][0] + 3), (0, 0, so["Q"][0] + 2 + nx)]
    base = dev[0]
    E = torch.zeros((len(idx),) + tuple(base.shape), dtype=torch.float64, device="cuda")
    for j, ix in enumerate(idx):
        E[(j,) + ix] = 1.0
    stage_of = lambda p: (base + torch.tensordot(p, E, dims=1)).contiguous()

    p0 = torch.zeros(len(idx), dtype=torch.float64, device="cuda")
    Jf = torch.func.jacfwd(lambda p: ag.lq_factor_fwd(s, stage_of(p), *rest, mu)[1][:, 0, :nu, :])(p0)
    Jr = torch.func.jacrev(lambda p: ag.lq_factor(s, stage_of(p), *rest, mu)[1][:, 0, :nu, :])(p0)
    assert Jf.shape == Jr.shape == (2, nu, nx, len(idx))
    assert gen.rel_fro(Jf.cpu().numpy(), Jr.cpu().numpy()) <= 1e-9
    assert float(Jf.abs().max()) > 0
    # backward through lq_factor_fwd raises, naming lq_factor
    st = dev[0].clone().requires_grad_()
    out = ag.lq_factor_fwd(s, st, *rest, mu)
    with pytest.raises(RuntimeError, match="lq_factor"):
        out[1].sum().backward()
    # vmap over the problem data raises
    with pytest.raises(NotImplementedError):
        torch.func.vmap(lambda x: ag.lq_factor_fwd(s, x, *rest, mu)[0])(dev[0][None].expand(2, *dev[0].shape)
                                                                         .contiguous())
    # the CPU oracle agrees with jacfwd on one column
    cpu_st = torch.tensor(recs[0])
    e = torch.zeros_like(cpu_st)
    e[idx[0]] = 1.0
    _, tK = torch.func.jvp(lambda x: adj.torch_factor(x, torch.tensor(recs[1]), case, mu)["fb"][:, 0, :nu, :], (cpu_st,),
                           (e,))
    assert gen.rel_fro(Jf[..., 0].cpu().numpy(), tK.numpy()) <= 1e-9
    s.close()
