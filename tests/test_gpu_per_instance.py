"""Per-instance penalty, regularisation and step length (the *_v twins of the C ABI, gar.h).

Every twin must give each instance exactly what the scalar call gives at that instance's value: the reference is
the scalar call run once per value on the whole batch, each instance's outputs taken from the run at its own value,
and the comparison is array equality."""
import numpy as np
import pytest

import gen

pytestmark = pytest.mark.gpu

MUS = (1.0, 1e-2, 1e-5)
OUTS_PLAIN = range(13)       # OUT_FF .. OUT_LBDAS
OUTS_PARAM = range(13, 20)   # OUT_FTH .. OUT_THHESS


@pytest.fixture(scope="module")
def gar():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import __graft_entry__ as g
    g.build()
    import aligator_b200.gar as gar
    return gar


def _records(gar, s, nx, nu, nc, nct, nc0, N, B, seed):
    """Stage / terminal records for handle `s` (parametric blocks, when the handle has them, small and random)."""
    probs = gen.generate_batch(seed, B, N, nx, nu, nc, nct)
    stage, term, G0, g0 = gar.pack_problems(probs)
    rec_nth = 0 if s.legs else s.nth
    if rec_nth:
        rng = np.random.default_rng(seed)
        plain = 2 * nx * nx + 2 * nx * nu + nu * nu + 2 * nx + nu + nc * (nx + nu + 1)
        st = np.zeros((B, N, s.srec))
        st[..., :plain] = stage.reshape(B, N, -1)[..., :plain]
        st[..., plain:plain + rec_nth * (nx + nu + nc + rec_nth + 1)] = 0.1 * rng.standard_normal(
            (B, N, rec_nth * (nx + nu + nc + rec_nth + 1)))
        tt = np.zeros((B, s.trec))
        tt[:, :term.shape[1]] = term
        tt[:, term.shape[1]:] = 0.1 * rng.standard_normal((B, s.trec - term.shape[1]))
        stage, term = st, tt
    return [np.ascontiguousarray(a) for a in (stage, term, G0, g0)]


def _outputs(gar, s):
    outs = list(OUTS_PLAIN) + (list(OUTS_PARAM) if s.nth else [])
    r = {w: s.get(w).copy() for w in outs if int(np.prod(s.out_shape(w)))}
    r["status"] = s.status().copy()
    return r


def _mu_per_instance(B):
    return np.array([MUS[b % 3] for b in range(B)])


def _expected(gar, s, mu_b, run):
    """Each instance's outputs from the scalar run at its own mu."""
    ref = {}
    for v in MUS:
        run(v)
        out = _outputs(gar, s)
        sel = mu_b == v
        for k, a in out.items():
            ref.setdefault(k, np.empty_like(a))[sel] = a[sel]
    return ref


def _assert_equal(got, want, tag=""):
    for k in want:
        assert np.array_equal(got[k], want[k], equal_nan=True), (tag, k)


# (name, CudaRiccatiBatch keyword arguments, (nx, nu, nc, nct, nc0, N, B))
HANDLES = [("lane_v%d" % v, dict(variant=v), (4, 2, 2, 2, 4, 9, 37)) for v in range(7)] + [
    ("lane_12_6_6", {}, (12, 6, 6, 3, 12, 7, 11))] + [
    ("mma_v%d" % v, dict(variant=v), (12, 6, 0, 3, 12, 8, 21)) for v in (6, 7, 8, 10)] + [
    ("mma_14_7_v7", dict(variant=7), (14, 7, 0, 2, 14, 5, 9)),
    ("cta_v9", dict(variant=9), (4, 2, 2, 2, 4, 9, 13)),
    ("cta_runtime", {}, (7, 3, 2, 2, 7, 6, 10)),
    ("parametric", dict(nth=2), (5, 2, 1, 1, 5, 5, 7)),
    ("legs", dict(legs=3), (4, 2, 2, 2, 4, 8, 9)),
    ("dense", dict(dense=True), (4, 2, 2, 2, 4, 6, 8)),
]


@pytest.mark.parametrize("name,kw,dims", HANDLES, ids=[h[0] for h in HANDLES])
def test_sweep_and_backward_v_match_scalar_runs(gar, name, kw, dims):
    import torch
    nx, nu, nc, nct, nc0, N, B = dims
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
    s.set_problem(*_records(gar, s, nx, nu, nc, nct, nc0, N, B, seed=nx * 100 + B))
    mu_b = _mu_per_instance(B)
    want = _expected(gar, s, mu_b, s.sweep)
    mu_d = torch.tensor(mu_b, device="cuda")
    n0 = s.launch_count()
    s.sweep(mu_d)                                       # device array
    s.synchronize()
    n1 = s.launch_count()
    got = _outputs(gar, s)
    _assert_equal(got, want, name + " sweep_v")
    s.backward(mu_b)                                    # host array, then a forward pass that reads no mu
    s.forward()
    _assert_equal(_outputs(gar, s), want, name + " backward_v + forward")
    s.sweep(MUS[0])
    s.sweep(mu_b)
    _assert_equal(_outputs(gar, s), want, name + " sweep_v (host)")
    n2 = s.launch_count()
    s.sweep(MUS[0])
    assert s.launch_count() - n2 == n1 - n0  # the twin launches what the scalar call launches
    if s.legs or not s.nth:  # kkt_error_v on every handle type kkt_error serves (not parametric records)
        s.sweep(mu_d)
        got_k = s.kkt_error(mu_d)
        want_k = np.empty_like(got_k)
        for v in MUS:
            s.sweep(v)
            want_k[mu_b == v] = s.kkt_error(v)[mu_b == v]
        assert np.array_equal(got_k, want_k, equal_nan=True), name + " kkt_error_v"
    s.close()


def _launches(s, call):
    n0 = s.launch_count()
    call()
    s.synchronize()
    return s.launch_count() - n0


@pytest.mark.parametrize("dims", [(4, 2, 2, 2, 4, 9, 37), (12, 6, 0, 3, 12, 8, 21)])
def test_launch_counts_guard_and_memory_spaces(gar, dims):
    import torch
    nx, nu, nc, nct, nc0, N, B = dims
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    recs = _records(gar, s, nx, nu, nc, nct, nc0, N, B, seed=7)
    for a in recs:  # instances 1 and 2 get the records of instance 0 (and mu = 1e-2, 1e-5 where 0 has 1)
        a[1:3] = a[0]
    s.set_problem(*recs)
    mu_b = _mu_per_instance(B)
    mu_d = torch.tensor(mu_b, device="cuda")
    assert _launches(s, lambda: s.sweep(mu_d)) == _launches(s, lambda: s.sweep(1.0))
    assert _launches(s, lambda: s.backward(mu_b)) == _launches(s, lambda: s.backward(1.0))
    s.sweep(mu_d)
    dev = _outputs(gar, s)
    s.sweep(mu_b)
    host = _outputs(gar, s)
    _assert_equal(host, dev, "host vs device mueq")
    # the guard: the same records at different mu differ where mu enters (Z = C / mu, z = d / mu, the multipliers),
    # which an array the kernels silently ignored would not give
    for w in (gar.OUT_FBT, gar.OUT_FFT, gar.OUT_VST) + ((gar.OUT_VS,) if nc else ()):
        a = dev[w]
        assert not np.array_equal(a[0], a[1]) and not np.array_equal(a[1], a[2]) and not np.array_equal(a[0], a[2]), w
    # ... and each equals the scalar run at its own mu
    for b, v in enumerate(MUS):
        s.sweep(v)
        assert all(np.array_equal(s.get(w)[b], dev[w][b]) for w in dev if w != "status"), v
    s.close()


def test_large_batch_two_rounds_and_ragged_tail(gar):
    """C2 dimensions with terminal constraints, 2200 instances: more than one round of resident CTAs on 132 SMs
    and a partly filled last CTA."""
    import torch
    nx, nu, nc, nct, nc0, N, B = 12, 6, 0, 3, 12, 6, 2200
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    s.set_problem(*_records(gar, s, nx, nu, nc, nct, nc0, N, B, seed=2200))
    info = s.kernel_info()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert info["grid"] > sms * info["ctas_per_sm"] and info["grid"] % (sms * info["ctas_per_sm"]) != 0
    mu_b = _mu_per_instance(B)
    want = _expected(gar, s, mu_b, s.sweep)
    s.sweep(torch.tensor(mu_b, device="cuda"))
    _assert_equal(_outputs(gar, s), want, "2200")
    s.close()


def test_call_order_leaves_no_trace(gar):
    import torch
    nx, nu, nc, nct, nc0, N, B = 4, 2, 2, 2, 4, 9, 37
    mu0 = 0.3
    a = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    recs = _records(gar, a, nx, nu, nc, nct, nc0, N, B, seed=11)
    a.set_problem(*recs)
    a.backward(torch.tensor(_mu_per_instance(B), device="cuda"))
    a.backward(mu0)
    a.forward()
    got = _outputs(gar, a)
    b = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    b.set_problem(*recs)
    b.backward(mu0)
    b.forward()
    _assert_equal(got, _outputs(gar, b), "scalar after _v")
    # kkt_error_v: each instance as the scalar call at its own mu
    mu_b = _mu_per_instance(B)
    a.sweep(torch.tensor(mu_b, device="cuda"))
    got = a.kkt_error(torch.tensor(mu_b, device="cuda"))
    want = np.empty_like(got)
    for v in MUS:
        b.sweep(v)
        k = b.kkt_error(v)
        want[mu_b == v] = k[mu_b == v]
    assert np.array_equal(got, want)
    a.close()
    b.close()


def test_invalid_mu(gar):
    import torch
    nx, nu, nc, nct, nc0, N, B = 4, 2, 2, 2, 4, 9, 37
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    s.set_problem(*_records(gar, s, nx, nu, nc, nct, nc0, N, B, seed=3))
    mu_b = _mu_per_instance(B)
    s.sweep(torch.tensor(mu_b, device="cuda"))
    clean = _outputs(gar, s)
    bad = mu_b.copy()
    bad[5], bad[17], bad[30] = np.nan, -1.0, 0.0
    s.sweep(torch.tensor(bad, device="cuda"))
    got = _outputs(gar, s)
    st = got["status"]
    assert np.all(st[[5, 17, 30]] & 8) and not np.any(np.delete(st, [5, 17, 30]))
    keep = np.setdiff1d(np.arange(B), [5, 17, 30])
    for k in clean:
        assert np.array_equal(got[k][keep], clean[k][keep], equal_nan=True), k
    n0 = s.launch_count()
    with pytest.raises(gar.GarError):
        s.sweep(bad)
    with pytest.raises(gar.GarError):
        s.backward(bad)
    assert s.launch_count() == n0
    with pytest.raises(ValueError):
        s.sweep(mu_b[:-1])
    with pytest.raises(ValueError):
        s.sweep(mu_b.astype(np.float32))
    s.close()


@pytest.mark.parametrize("dims", [(4, 2, 2, 2, 4, 9, 37), (12, 6, 0, 3, 12, 8, 21)])
def test_host_sweeps(gar, dims):
    import torch
    nx, nu, nc, nct, nc0, N, B = dims
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    recs = _records(gar, s, nx, nu, nc, nct, nc0, N, B, seed=5)
    s.set_problem(*recs)
    mu_b = _mu_per_instance(B)
    s.sweep(torch.tensor(mu_b, device="cuda"))
    want = _outputs(gar, s)
    sym = s.pack_stage_sym(recs[0])
    for nchunks in (1, 3):
        for which in ("full", "sym"):
            outs = {w: np.empty(int(np.prod(s.out_shape(w)))) for w in OUTS_PLAIN if int(np.prod(s.out_shape(w)))}
            if which == "full":
                s.sweep_host(recs[0], recs[1], recs[2], recs[3], mu_b, outs, nchunks=nchunks)
            else:
                s.sweep_host_sym(sym, recs[1], recs[2], recs[3], mu_b, outs, nchunks=nchunks)
            s.synchronize()
            got = _outputs(gar, s)
            _assert_equal(got, want, (which, nchunks))
            for w, a in outs.items():
                g = s.get(w)
                assert np.array_equal(a.reshape(s.out_shape(w)), g if w not in (gar.OUT_VXX,) else g.transpose(0, 1, 3, 2)), w
    s.close()


def _rand_dev(torch, g, *shape):
    return torch.randn(*shape, generator=g, device="cuda", dtype=torch.float64)


def test_streaming_twins(gar):
    """linear_step_v, al_value_v, multipliers_v, assemble_v, fddp_backward_pass_v against per-group scalar calls."""
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    nx, nu, nc, nct, nc0, N, B = 4, 2, 2, 2, 4, 7, 30
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    s.set_problem(*_records(gar, s, nx, nu, nc, nct, nc0, N, B, seed=9))
    s.sweep(0.1)
    grp = np.arange(B) % 3
    rd = lambda *sh: _rand_dev(torch, g, B, *sh)
    cur = dict(xs=rd(N + 1, nx), us=rd(N, nu), vs=rd(N, nc), vsT=rd(nct), lam0=rd(nc0), lams=rd(N, nx))
    # linear step: alpha in {0, 0.5, 1}
    alphas = (0.0, 0.5, 1.0)
    al = np.array([alphas[k] for k in grp])
    trial = {k: torch.empty_like(v) for k, v in cur.items()}
    s.linear_step(torch.tensor(al, device="cuda"), cur, trial)
    s.synchronize()
    for k in cur:
        assert torch.equal(trial[k][torch.tensor(al == 0.0, device="cuda")], cur[k][torch.tensor(al == 0.0, device="cuda")])
    for j, a in enumerate(alphas):
        ref = {k: torch.empty_like(v) for k, v in cur.items()}
        s.linear_step(a, cur, ref)
        s.synchronize()
        sel = torch.tensor(grp == j, device="cuda")
        for k in cur:
            assert torch.equal(trial[k][sel], ref[k][sel]), (k, a)
    # AL value and multipliers at per-instance mu, mu_dyn = 0.1 mu
    mu_b = _mu_per_instance(B)
    mud_b = 0.1 * mu_b
    cost = rd()
    got = s.al_value(cur, cost, torch.tensor(mud_b, device="cuda"), torch.tensor(mu_b, device="cuda"))
    want = np.empty(B)
    for v in MUS:
        want[mu_b == v] = s.al_value(cur, cost, 0.1 * v, v)[mu_b == v]
    assert np.array_equal(got, want)
    inp = dict(xs=cur["xs"], lam0=cur["lam0"], lams=cur["lams"], vs=cur["vs"], vsT=cur["vsT"], prev_vs=rd(N, nc),
               prev_vsT=rd(nct), init_value=rd(nc0), xnext=rd(N, nx), cval=rd(N, nc), cval_N=rd(nct),
               lo=torch.tensor([-np.inf, -0.5], device="cuda"), hi=torch.tensor([0.0, 0.5], device="cuda"),
               loN=torch.tensor([np.inf, -np.inf], device="cuda"), hiN=torch.tensor([np.inf, 0.0], device="cuda"))
    e = lambda *sh: torch.empty(B, *sh, device="cuda", dtype=torch.float64)
    mk = lambda: dict(slack=e(N, nx), lam0_plus=e(nc0), lams_plus=e(N, nx), vs_plus=e(N, nc), vsT_plus=e(nct),
                      shifted=e(N, nc), shifted_N=e(nct), Lv=e(N, nc), Lv_N=e(nct))
    o = mk()
    sc = s.multipliers(inp, o, torch.tensor(mu_b, device="cuda"), mud_b)
    for v in MUS:
        r = mk()
        scr = s.multipliers(inp, r, v, 0.1 * v)
        sel = mu_b == v
        assert np.array_equal(sc[sel], scr[sel])
        for k in o:
            assert torch.equal(o[k][torch.tensor(sel, device="cuda")], r[k][torch.tensor(sel, device="cuda")]), k
    # assembly with per-instance preg and mu_inv = 1 / mu
    pregs = (1e-8, 1e-4, 1e-1)
    preg_b = np.array([pregs[k] for k in grp])
    cm = lambda *sh: rd(*sh)
    lq = dict(Jx=cm(N, nx * nx), Ju=cm(N, nx * nu), slack=o["slack"], Lxx=cm(N, nx * nx), Lxu=cm(N, nx * nu),
              Luu=cm(N, nu * nu), Lx=cm(N, nx), Lu=cm(N, nu), cJx=cm(N, nc * nx), cJu=cm(N, nc * nu), Lv=o["Lv"],
              shifted=o["shifted"], lo=inp["lo"], hi=inp["hi"], Lxx_N=cm(nx * nx), Lx_N=cm(nx), cJx_N=cm(nct * nx),
              Lv_N=o["Lv_N"], shifted_N=o["shifted_N"], loN=inp["loN"], hiN=inp["hiN"], G0=cm(nc0 * nx), g0=cm(nc0))
    s.assemble(lq, torch.tensor(preg_b, device="cuda"), torch.tensor(1.0 / mu_b, device="cuda"))
    got = [s.get_problem(w).reshape(B, -1) for w in range(4)]
    for j, p in enumerate(pregs):
        for v in MUS:
            sel = (grp == j) & (mu_b == v)
            if not sel.any():
                continue
            s.assemble(lq, p, 1.0 / v)
            for w in range(4):
                assert np.array_equal(got[w][sel], s.get_problem(w).reshape(B, -1)[sel]), (w, p, v)
    s.close()
    # FDDP backward pass with per-instance preg
    nx, nu, N = 6, 3, 5
    f = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B)
    rng = np.random.default_rng(2)
    spd = lambda n: (lambda W: W @ np.swapaxes(W, -1, -2) / n + np.eye(n))(rng.standard_normal((B, N, n, n)))
    T = lambda a: torch.tensor(np.ascontiguousarray(a), device="cuda")
    H = spd(nx + nu)
    arr = dict(Jx=T(np.eye(nx) + 0.1 * rng.standard_normal((B, N, nx, nx))), Ju=T(rng.standard_normal((B, N, nx, nu))),
               fs=T(0.1 * rng.standard_normal((B, N + 1, nx))), Lxx=T(H[..., :nx, :nx]), Lxu=T(H[..., :nx, nx:]),
               Luu=T(H[..., nx:, nx:]), Lx=T(rng.standard_normal((B, N, nx))), Lu=T(rng.standard_normal((B, N, nu))),
               Lxx_N=T(spd(nx)[:, 0]), Lx_N=T(rng.standard_normal((B, nx))))
    Vx, Qk = torch.empty(B, N + 1, nx, device="cuda", dtype=torch.float64), torch.empty(B, N, nu, device="cuda", dtype=torch.float64)
    f.fddp_backward_pass(arr, torch.tensor(preg_b, device="cuda"), Vx, Qk)
    f.synchronize()
    got = dict(Vx=Vx.cpu().numpy(), Qk=Qk.cpu().numpy(), ff=f.get(gar.OUT_FF).copy(), fb=f.get(gar.OUT_FB).copy(),
               Vxx=f.get(gar.OUT_VXX).copy())
    for j, p in enumerate(pregs):
        f.fddp_backward_pass(arr, p, Vx, Qk)
        f.synchronize()
        ref = dict(Vx=Vx.cpu().numpy(), Qk=Qk.cpu().numpy(), ff=f.get(gar.OUT_FF), fb=f.get(gar.OUT_FB),
                   Vxx=f.get(gar.OUT_VXX))
        sel = grp == j
        for k in got:
            assert np.array_equal(got[k][sel], ref[k][sel]), (k, p)
    f.close()


@pytest.mark.parametrize("dims", [(4, 2, 2, 0, 4, 100, 16384), (5, 2, 2, 2, 5, 20, 300)], ids=["c3", "nc2_nct2"])
def test_whole_inner_iteration_matches_per_group_scalar_chains(gar, dims):
    """One inner iteration chained on the device as in INTEGRATION 3b -- multipliers_v -> al_value_v -> assemble_v ->
    sweep_v -> linear_step_v with per-instance mu, mu_dyn = 0.1 mu, preg and alpha -- against the same chain of scalar
    calls run once per group of instances that share their values: every array, bit for bit."""
    import torch
    nx, nu, nc, nct, nc0, N, B = dims
    g = torch.Generator(device="cuda")
    g.manual_seed(B)
    rd = lambda *sh: _rand_dev(torch, g, B, *sh)
    spd = lambda n, *lead: (lambda M: (M @ M.transpose(-1, -2) / n + torch.eye(n, dtype=torch.float64, device="cuda"))
                            .reshape(B, *lead, n * n))(rd(*lead, n, n))
    cur = dict(xs=rd(N + 1, nx), us=rd(N, nu), vs=rd(N, nc), vsT=rd(nct), lam0=rd(nc0), lams=rd(N, nx))
    lo = torch.tensor([[float("inf"), -float("inf"), -0.5][i % 3] for i in range(max(nc, nct))], device="cuda",
                      dtype=torch.float64)
    hi = torch.tensor([[float("inf"), 0.0, 0.5][i % 3] for i in range(max(nc, nct))], device="cuda", dtype=torch.float64)
    inp = dict(xs=cur["xs"], lam0=cur["lam0"], lams=cur["lams"], vs=cur["vs"], vsT=cur["vsT"], prev_vs=rd(N, nc),
               prev_vsT=rd(nct), init_value=rd(nc0), xnext=rd(N, nx), cval=rd(N, nc), cval_N=rd(nct), lo=lo[:nc],
               hi=hi[:nc], loN=lo[:nct], hiN=hi[:nct])
    model = dict(Jx=0.3 * rd(N, nx * nx), Ju=rd(N, nx * nu), Lxx=spd(nx, N), Lxu=0.1 * rd(N, nx * nu), Luu=spd(nu, N),
                 Lx=rd(N, nx), Lu=rd(N, nu), cJx=rd(N, nc * nx), cJu=rd(N, nc * nu), Lxx_N=spd(nx), Lx_N=rd(nx),
                 cJx_N=rd(nct * nx), G0=rd(nc0 * nx), cost=rd())
    grp = np.arange(B) % 3
    mus, pregs, alphas = (1e-1, 1e-2, 1e-3), (1e-8, 1e-5, 1e-2), (1.0, 0.5, 0.25)
    vals = lambda t: np.array([t[k] for k in grp])
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    e = lambda *sh: torch.empty(B, *sh, device="cuda", dtype=torch.float64)

    def chain(mu, mu_dyn, mu_inv, preg, alpha):
        o = dict(slack=e(N, nx), lam0_plus=e(nc0), lams_plus=e(N, nx), vs_plus=e(N, nc), vsT_plus=e(nct),
                 shifted=e(N, nc), shifted_N=e(nct), Lv=e(N, nc), Lv_N=e(nct))
        sc = e(2)
        s.multipliers(inp, o, mu, mu_dyn, out=sc)
        plus = dict(lam0=o["lam0_plus"], lams=o["lams_plus"], vs=o["vs_plus"], vsT=o["vsT_plus"])
        phi = s.al_value(plus, model["cost"], mu_dyn, mu)
        s.assemble(dict(Jx=model["Jx"], Ju=model["Ju"], slack=o["slack"], Lxx=model["Lxx"], Lxu=model["Lxu"],
                        Luu=model["Luu"], Lx=model["Lx"], Lu=model["Lu"], cJx=model["cJx"], cJu=model["cJu"], Lv=o["Lv"],
                        shifted=o["shifted"], lo=inp["lo"], hi=inp["hi"], Lxx_N=model["Lxx_N"], Lx_N=model["Lx_N"],
                        cJx_N=model["cJx_N"], Lv_N=o["Lv_N"], shifted_N=o["shifted_N"], loN=inp["loN"],
                        hiN=inp["hiN"], G0=model["G0"], g0=inp["init_value"]), preg, mu_inv)
        s.sweep(mu)
        trial = {k: torch.empty_like(v) for k, v in cur.items()}
        s.linear_step(alpha, cur, trial)
        s.synchronize()
        r = {k: v.cpu().numpy() for k, v in o.items()}
        r.update({"trial_" + k: v.cpu().numpy() for k, v in trial.items()})
        r.update(sc=sc.cpu().numpy(), phi=phi, stage=s.get_problem(0).reshape(B, -1), term=s.get_problem(1).reshape(B, -1))
        r.update({"out%d" % w: s.get(w).copy() for w in OUTS_PLAIN if int(np.prod(s.out_shape(w)))})
        r["status"] = s.status().copy()
        return r

    T = lambda a: torch.tensor(a, device="cuda")
    mu_b = vals(mus)
    got = chain(T(mu_b), T(0.1 * mu_b), T(1.0 / mu_b), T(vals(pregs)), T(vals(alphas)))
    assert np.all(got["status"] == 0)
    for j in range(3):
        ref = chain(mus[j], 0.1 * mus[j], 1.0 / mus[j], pregs[j], alphas[j])
        sel = grp == j
        for k in ref:
            if ref[k].shape and ref[k].shape[0] == B:
                assert np.array_equal(got[k][sel], ref[k][sel], equal_nan=True), (k, j)
    s.close()
