"""Multiplier estimates, Lagrangian gradients and stopping criteria of SolverProxDDP's inner iteration
(computeMultipliers, solver-proxddp.hxx:220-318; LagrangianDerivatives::compute, core/lagrangian.hpp:29-92;
computeCriterion, solver-proxddp.hxx:703-732).  CPU: the numpy restatement against hand-computed numbers and
against a dense formulation of the Lagrangian.  GPU: ab2_gar_multipliers, ab2_gar_lagrangian_gradient and
ab2_gar_criterion against the restatement, and one whole inner iteration chained on the device against the same
chain built from the restatements."""
import numpy as np
import pytest

import gen
from oracle import proxddp_inner as pin

INF = np.inf


# ---------------------------------------------------------------------------------------------------------------
# CPU: the restatement
# ---------------------------------------------------------------------------------------------------------------
def _hand_case():
    """nx = 2, nu = 1, nc = 3 (equality, negative orthant, box [-1, 1]), nct = 1 (negative orthant), nc0 = 2, N = 1.
    Every number is dyadic, so each expected value below is exact."""
    return dict(
        xs=[np.array([1.0, 2.0]), np.array([3.0, -1.0])],
        lams=[np.array([1.0, -1.0]), np.array([2.0, 0.0])],
        vs=[np.array([1.0, 2.0, -1.0]), np.array([3.0])],
        prev_vs=[np.array([0.5, 1.0, 1.0]), np.array([0.5])],
        init_value=np.array([0.5, -0.5]),
        cvals=[np.array([0.25, 0.0, 0.5]), np.array([-1.0])],
        lo=np.array([INF, -INF, -1.0]), hi=np.array([INF, 0.0, 1.0]), loN=np.array([-INF]), hiN=np.array([0.0]),
        mu=0.5, mu_dyn=0.25, xnext=[np.array([13.0, 9.0])])


def test_multipliers_hand_case():
    h = _hand_case()
    m = pin.compute_multipliers(**h)
    assert np.array_equal(m["fs"][0], [0.5, -0.5]) and np.array_equal(m["fs"][1], [10.0, 10.0])  # xnext - x1
    # lam0_plus = lam0 + fs0 / mu (mu = 0.5; with mu_dyn it would be [3, -3])
    assert np.array_equal(m["lams_plus"][0], [2.0, -2.0])
    assert np.array_equal(m["lams_plus"][1], [42.0, 40.0])  # lam1 + fs1 / mu_dyn
    # shifted = cval + mu prev = [0.5, 0.5, 1.0]: the box row sits exactly ON its upper bound
    assert np.array_equal(m["shifted"][0], [0.5, 0.5, 1.0])
    # NC = [0.5 (equality: z), max(0.5, 0) = 0.5, 1 - clamp(1, -1, 1) = 0 (on the bound: not outside)]
    assert np.array_equal(m["vs_plus"][0], [1.0, 1.0, 0.0])            # NC / mu
    assert np.array_equal(m["Lvs"][0], [0.0, -0.5, 0.5])               # NC - mu vs
    assert np.array_equal(m["stage_infeas"][0], [0.25, 0.0, -0.5])     # mu (vs_plus - prev)
    # terminal: shifted = -1 + 0.25 = -0.75 < 0: projection 0
    assert np.array_equal(m["shifted"][1], [-0.75]) and np.array_equal(m["vs_plus"][1], [0.0])
    assert np.array_equal(m["Lvs"][1], [-1.5]) and np.array_equal(m["stage_infeas"][1], [-0.25])
    assert m["prim_infeas"] == 10.0 and m["ok"]  # fs_N = fs_1 counts in the primal infeasibility
    # the same with the dynamics residual given directly
    h2 = dict(h, xnext=None, fs=[np.array([10.0, 10.0])])
    m2 = pin.compute_multipliers(**h2)
    for k in ("lams_plus", "vs_plus", "Lvs", "shifted"):
        assert all(np.array_equal(a, b) for a, b in zip(m[k], m2[k]))
    # a NaN anywhere upstream of lams_plus / Lvs clears the flag
    h3 = dict(h, cvals=[np.array([0.25, np.nan, 0.5]), np.array([-1.0])])
    assert not pin.compute_multipliers(**h3)["ok"]


def _hand_gradient_inputs():
    return dict(lx=[np.array([0.5, 0.5])], lu=[np.array([1.0])], lx_N=np.array([1.0, 1.0]),
                Jx=[np.array([[1.0, 2.0], [3.0, 4.0]])], Ju=[np.array([[1.0], [5.0]])],
                cJx=[np.array([[1.0, 0.0], [0.0, 1.0], [1.0, 1.0]])], cJu=[np.array([[0.0], [1.0], [2.0]])],
                cJx_N=np.array([[2.0, -1.0]]), G0=np.array([[1.0, 0.0], [0.0, 2.0]]))


def test_gradient_and_criterion_hand_case():
    h = _hand_case()
    g = _hand_gradient_inputs()
    Lxs, Lus = pin.lagrangian_gradient(**g, lams=h["lams"], vs=h["vs"])
    # Lx_0 = G0^T lam0 (1, -2) + lx (0.5, 0.5) + Jx^T lam1 (2, 4) + cJx^T v0 (0, 1)
    assert np.array_equal(Lxs[0], [3.5, 3.5])
    assert np.array_equal(Lus[0], [3.0])          # lu 1 + Ju^T lam1 2 + cJu^T v0 0
    assert np.array_equal(Lxs[1], [5.0, -2.0])    # -lam1 (-2, 0) + lx_N (1, 1) + cJx_N^T vN (6, -3)
    Lxs_f, _ = pin.lagrangian_gradient(**g, lams=h["lams"], vs=h["vs"], force_initial_condition=True)
    assert np.array_equal(Lxs_f[0], [0.0, 0.0]) and np.array_equal(Lxs_f[1], Lxs[1])
    m = pin.compute_multipliers(**h)
    crit, dual = pin.criterion(Lxs, Lus, m["fs"], m["Lvs"])
    # stage 0: max(3.5, 3, |fs0| 0.5, |Lv0| 0.5); terminal: max(5, |Lv_N| 1.5).  fs_N = (10, 10) is NOT counted.
    assert crit == 5.0 and dual == 5.0
    fs = [np.array([0.5, -7.0]), m["fs"][1]]      # fs0 IS counted (stage 0's residual)
    assert pin.criterion(Lxs, Lus, fs, m["Lvs"]) == (7.0, 5.0)
    # N = 0: the only knot is the terminal one, Lx_0 = G0^T lam0 + lx_N + cJx_N^T vN; no dynamics residual counts
    L0, _ = pin.lagrangian_gradient([], [], g["lx_N"], [], [], [], [], g["cJx_N"], g["G0"], [h["lams"][0]], [h["vs"][1]])
    assert np.array_equal(L0[0], [1.0 + 1.0 + 6.0, -2.0 + 1.0 - 3.0])
    assert pin.criterion(L0, [], [np.array([100.0, 0.0])], [np.array([-1.5])]) == (8.0, 8.0)


def _random_instance(rng, N, nx, nu, nc, nct, nc0):
    r = lambda *s: rng.standard_normal(s)
    return dict(lx=list(r(N, nx)), lu=list(r(N, nu)), lx_N=r(nx), Jx=list(r(N, nx, nx)), Ju=list(r(N, nx, nu)),
                cJx=list(r(N, nc, nx)), cJu=list(r(N, nc, nu)), cJx_N=r(nct, nx), G0=r(nc0, nx)), \
        [r(nc0)] + list(r(N, nx)), list(r(N, nc)) + [r(nct)]


@pytest.mark.parametrize("dims", [(3, 3, 2, 2, 1, 3), (4, 5, 3, 0, 2, 2), (0, 4, 2, 0, 3, 4)])
def test_gradient_oracle_matches_dense_lagrangian(dims):
    """Independent check: every constraint Jacobian of the instance stacked into ONE dense matrix J (initial
    condition, dynamics [Jx Ju -I], path constraints, terminal constraints) over z = (x0, u0, ..., x_N); then
    grad cost + J^T y from one dense mat-vec must equal the per-knot restatement."""
    N, nx, nu, nc, nct, nc0 = dims
    rng = np.random.default_rng(sum(dims))
    g, lams, vs = _random_instance(rng, N, nx, nu, nc, nct, nc0)
    nz = N * (nx + nu) + nx
    xo = lambda t: t * (nx + nu)
    rows, ys = [], []
    Jr = np.zeros((nc0, nz))
    Jr[:, :nx] = g["G0"]
    rows.append(Jr), ys.append(lams[0])
    for t in range(N):
        D = np.zeros((nx, nz))
        D[:, xo(t):xo(t) + nx], D[:, xo(t) + nx:xo(t + 1)] = g["Jx"][t], g["Ju"][t]
        D[:, xo(t + 1):xo(t + 1) + nx] = -np.eye(nx)
        P = np.zeros((nc, nz))
        P[:, xo(t):xo(t) + nx], P[:, xo(t) + nx:xo(t + 1)] = g["cJx"][t], g["cJu"][t]
        rows += [D, P]
        ys += [lams[t + 1], vs[t]]
    T = np.zeros((nct, nz))
    T[:, xo(N):] = g["cJx_N"]
    rows.append(T), ys.append(vs[N])
    grad = np.concatenate([np.concatenate([g["lx"][t], g["lu"][t]]) for t in range(N)] + [g["lx_N"]])
    dense = grad + np.vstack(rows).T @ np.concatenate(ys)
    Lxs, Lus = pin.lagrangian_gradient(**g, lams=lams, vs=vs)
    mine = np.concatenate([np.concatenate([Lxs[t], Lus[t]]) for t in range(N)] + [Lxs[N]])
    assert np.max(np.abs(mine - dense)) <= 1e-13 * max(1.0, np.max(np.abs(dense)))


# ---------------------------------------------------------------------------------------------------------------
# GPU: the device entry points against the restatement
# ---------------------------------------------------------------------------------------------------------------
def _bounds(n, kinds):
    lo = np.where(kinds == 0, INF, np.where(kinds == 1, -INF, -0.5))
    hi = np.where(kinds == 0, INF, np.where(kinds == 1, 0.0, 0.5))
    return lo, hi


def _device_inputs(torch, shape, seed):
    """Random inputs generated on the device.  Matrices are kept twice: `mat` [.., rows, cols] (for the host
    restatement) and their column-major device layout in `dev`."""
    N, nx, nu, nc, nct, nc0, B = shape
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device="cuda", dtype=torch.float64)
    mat = dict(Jx=rn(B, N, nx, nx), Ju=rn(B, N, nx, nu), cJx=rn(B, N, nc, nx), cJu=rn(B, N, nc, nu),
               cJx_N=rn(B, nct, nx), G0=rn(B, nc0, nx))
    dev = {k: v.transpose(-1, -2).contiguous() for k, v in mat.items()}
    vec = dict(xs=rn(B, N + 1, nx), lam0=rn(B, nc0), lams=rn(B, N, nx), vs=rn(B, N, nc), vsT=rn(B, nct),
               prev_vs=rn(B, N, nc), prev_vsT=rn(B, nct), init_value=rn(B, nc0), xnext=rn(B, N, nx),
               cval=rn(B, N, nc), cval_N=rn(B, nct), lx=rn(B, N, nx), lu=rn(B, N, nu), lx_N=rn(B, nx))
    dev.update(vec)
    rng = np.random.default_rng(seed)
    kinds = np.arange(nc) % 3  # equality, negative orthant, box rows mixed
    kindsN = (np.arange(nct) + 1) % 3
    rng.shuffle(kinds), rng.shuffle(kindsN)
    lo, hi = _bounds(nc, kinds)
    loN, hiN = _bounds(nct, kindsN)
    for k, v in dict(lo=lo, hi=hi, loN=loN, hiN=hiN).items():
        dev[k] = torch.tensor(v, device="cuda", dtype=torch.float64)
    return mat, dev


def _host(t, idx):
    import torch
    return t[torch.as_tensor(idx, device=t.device)].cpu().numpy() if t.numel() else np.zeros((len(idx),) + tuple(t.shape[1:]))


def _rel(a, b):
    return gen.rel_fro(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(5, 12, 6, 0, 0, 12, 7), (6, 4, 2, 2, 3, 4, 33), (3, 7, 3, 5, 0, 0, 5),
                                   (0, 4, 2, 0, 2, 4, 3), (4, 57, 28, 0, 0, 57, 2), (100, 12, 6, 0, 0, 12, 4096)])
def test_device_inner_matches_restatement(shape):
    import torch
    assert torch.cuda.is_available()
    import __graft_entry__ as gent
    gent.build()
    import aligator_b200.gar as gar
    N, nx, nu, nc, nct, nc0, B = shape
    mat, dev = _device_inputs(torch, shape, seed=sum(shape))
    bnan = B // 2  # this instance gets a NaN in its dynamics residual (or initial residual when N = 0)
    if N > 0:
        dev["xnext"][bnan, N // 2, nx // 2] = float("nan")
    else:
        dev["init_value"][bnan, 0] = float("nan")
    idx = np.arange(B) if B <= 64 else np.unique(np.linspace(0, B - 1, 64).astype(int))
    assert bnan in idx or B > 64
    if B > 64:
        idx = np.unique(np.append(idx, bnan))
    h = {k: _host(v, idx) for k, v in dev.items() if k not in ("lo", "hi", "loN", "hiN")}
    hm = {k: _host(v, idx) for k, v in mat.items()}
    bnd = {k: dev[k].cpu().numpy() for k in ("lo", "hi", "loN", "hiN")}
    mu, mu_dyn = 0.03, 0.007
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    e = lambda *sh: torch.empty(*sh, device="cuda", dtype=torch.float64)
    fs_dev = dev["xnext"] - dev["xs"][:, 1:]
    for mode in ("xnext", "fs"):
        out = dict(slack=e(B, N, nx), lam0_plus=e(B, nc0), lams_plus=e(B, N, nx), vs_plus=e(B, N, nc),
                   vsT_plus=e(B, nct), shifted=e(B, N, nc), shifted_N=e(B, nct), Lv=e(B, N, nc), Lv_N=e(B, nct))
        inp = {k: dev[k] for k in ("xs", "lam0", "lams", "vs", "vsT", "prev_vs", "prev_vsT", "init_value", "cval",
                                   "cval_N", "lo", "hi", "loN", "hiN")}
        if mode == "xnext":
            inp["xnext"] = dev["xnext"]
            sc = s.multipliers(inp, out, mu, mu_dyn)                   # host destination
        else:
            inp["fs"] = fs_dev
            sc_d = e(B, 2)
            s.multipliers(inp, out, mu, mu_dyn, out=sc_d)             # device destination
            sc = sc_d.cpu().numpy()
        torch.cuda.synchronize()
        got = {k: _host(v, idx) for k, v in out.items()}
        flags_ref = []
        for j, b in enumerate(idx):
            m = pin.compute_multipliers(
                list(h["xs"][j]), [h["lam0"][j]] + list(h["lams"][j]), list(h["vs"][j]) + [h["vsT"][j]],
                list(h["prev_vs"][j]) + [h["prev_vsT"][j]], h["init_value"][j],
                list(h["cval"][j]) + [h["cval_N"][j]], bnd["lo"], bnd["hi"], bnd["loN"], bnd["hiN"], mu, mu_dyn,
                xnext=list(h["xnext"][j]))
            flags_ref.append(m["ok"])
            assert sc[b, 1] == (1.0 if m["ok"] else 0.0), (mode, b)
            # the copy / difference is exact
            assert np.array_equal(got["slack"][j], np.array(m["fs"][1:]).reshape(N, nx), equal_nan=True)
            if b == bnan:
                continue
            assert _rel(got["lam0_plus"][j], m["lams_plus"][0]) <= 1e-15
            assert _rel(got["lams_plus"][j], np.array(m["lams_plus"][1:]).reshape(N, nx)) <= 1e-15
            stg = lambda key: np.array(m[key][:N]).reshape(N, nc)
            assert _rel(got["shifted"][j], stg("shifted")) <= 1e-15
            assert _rel(got["Lv"][j], stg("Lvs")) <= 1e-15
            assert _rel(got["vs_plus"][j], stg("vs_plus")) <= 1e-15
            # the projection itself (min / max, equality and active-set decisions) is exact on the device's shifted
            assert np.array_equal(got["vs_plus"][j], (1.0 / mu) * pin.normal_cone(got["shifted"][j], bnd["lo"], bnd["hi"]))
            assert np.array_equal(got["vsT_plus"][j], (1.0 / mu) * pin.normal_cone(got["shifted_N"][j], bnd["loN"], bnd["hiN"]))
            if nct:
                assert _rel(got["shifted_N"][j], m["shifted"][N]) <= 1e-15
                assert _rel(got["Lv_N"][j], m["Lvs"][N]) <= 1e-15
                assert _rel(got["vsT_plus"][j], m["vs_plus"][N]) <= 1e-15
            assert abs(sc[b, 0] - m["prim_infeas"]) <= 1e-13 * m["prim_infeas"]
        assert not flags_ref[list(idx).index(bnan)]
    # ---- Lagrangian gradient: both layouts, force_initial_condition off and on ----
    lag_in = {k: dev[k] for k in ("lx", "lu", "lx_N", "Jx", "Ju", "cJx", "cJu", "cJx_N", "G0", "lam0", "lams", "vs", "vsT")}
    for force in (False, True):
        lg = dict(Lx=e(B, N, nx), Lx_N=e(B, nx), Lu=e(B, N, nu), Lxs=e(B, N + 1, nx), Lus=e(B, N, nu))
        s.lagrangian_gradient(lag_in, lg, force_initial_condition=force)
        torch.cuda.synchronize()
        got = {k: _host(v, idx) for k, v in lg.items()}
        for j, b in enumerate(idx):
            Lxs, Lus = pin.lagrangian_gradient(
                list(h["lx"][j]), list(h["lu"][j]), h["lx_N"][j], list(hm["Jx"][j]), list(hm["Ju"][j]),
                list(hm["cJx"][j]), list(hm["cJu"][j]), hm["cJx_N"][j], hm["G0"][j],
                [h["lam0"][j]] + list(h["lams"][j]), list(h["vs"][j]) + [h["vsT"][j]], force_initial_condition=force)
            wx, wu = np.array(Lxs), np.array(Lus).reshape(N, nu)
            sx = max(1.0, np.max(np.abs(wx)))
            assert np.max(np.abs(got["Lxs"][j] - wx)) <= 1e-13 * sx, (force, b)
            if N:
                assert np.max(np.abs(got["Lus"][j] - wu)) <= 1e-13 * max(1.0, np.max(np.abs(wu)))
            # the assemble layout holds the same numbers
            assert np.array_equal(got["Lx"][j], got["Lxs"][j][:N]) and np.array_equal(got["Lx_N"][j], got["Lxs"][j][N])
            assert np.array_equal(got["Lu"][j], got["Lus"][j])
            if force:
                assert not np.any(got["Lxs"][j][0])
    # ---- criterion on the device's own arrays (force on, as innerLoop computes it) ----
    crit_in = dict(Lxs=lg["Lxs"], Lus=lg["Lus"], init_value=dev["init_value"], slack=out["slack"], Lv=out["Lv"],
                   Lv_N=out["Lv_N"])
    ch = s.criterion(crit_in)
    cd = e(B, 2)
    s.criterion(crit_in, out=cd)
    assert np.array_equal(cd.cpu().numpy(), ch, equal_nan=True)
    gc = {k: _host(v, idx) for k, v in crit_in.items()}
    for j, b in enumerate(idx):
        if b == bnan:
            continue
        fs = [gc["init_value"][j]] + list(gc["slack"][j])
        Lvs = list(gc["Lv"][j]) + [gc["Lv_N"][j]]
        ref = pin.criterion(list(gc["Lxs"][j]), list(gc["Lus"][j]), fs, Lvs)
        assert tuple(ch[b]) == ref, b  # maxima of the same numbers: exact
    s.close()


# ---------------------------------------------------------------------------------------------------------------
# GPU: one inner iteration chained on the device
# ---------------------------------------------------------------------------------------------------------------
class _LqModel:
    """A batched linear-quadratic OCP with box-constrained controls: x' = A x + B u + c, cost sum 1/2 x'Qx + q'x +
    1/2 u'Ru + r'u + terminal 1/2 x'Qn x + qn'x, u in [-1, 1], initial condition x0 - xinit = 0.  `xp` is torch or
    numpy; every evaluation is the same arithmetic in both."""

    def __init__(self, rng, B, N, nx, nu):
        spd = lambda *s: (lambda W: W @ np.swapaxes(W, -1, -2) / s[-1] + np.eye(s[-1]))(rng.standard_normal(s))
        self.A = np.eye(nx) + 0.2 * rng.standard_normal((B, N, nx, nx))
        self.B = rng.standard_normal((B, N, nx, nu))
        self.c = rng.standard_normal((B, N, nx))
        self.Q, self.R, self.Qn = spd(B, N, nx, nx), spd(B, N, nu, nu), spd(B, nx, nx)
        self.q, self.r, self.qn = rng.standard_normal((B, N, nx)), rng.standard_normal((B, N, nu)), rng.standard_normal((B, nx))
        self.xinit = rng.standard_normal((B, nx))
        self.N, self.nx, self.nu = N, nx, nu

    def on(self, conv):
        m = object.__new__(_LqModel)
        m.__dict__.update({k: (conv(v) if isinstance(v, np.ndarray) else v) for k, v in self.__dict__.items()})
        return m

    def evaluate(self, xs, us):
        mv = lambda M, v: (M @ v[..., None])[..., 0]
        x, xN = xs[:, :-1], xs[:, -1]
        xnext = mv(self.A, x) + mv(self.B, us) + self.c
        lx, lu, lxN = mv(self.Q, x) + self.q, mv(self.R, us) + self.r, mv(self.Qn, xN) + self.qn
        cost = (0.5 * (x * mv(self.Q, x)).sum((1, 2)) + (self.q * x).sum((1, 2)) + 0.5 * (us * mv(self.R, us)).sum((1, 2))
                + (self.r * us).sum((1, 2)) + 0.5 * (xN * mv(self.Qn, xN)).sum(1) + (self.qn * xN).sum(1))
        return dict(xnext=xnext, lx=lx, lu=lu, lx_N=lxN, cost=cost, cval=us, init_value=xs[:, 0] - self.xinit)


@pytest.mark.gpu
def test_one_inner_iteration_on_device_matches_restatement_chain():
    """multipliers -> al_value -> lagrangian_gradient(iterate) -> criterion -> assemble -> sweep ->
    lagrangian_gradient(plus) -> directional_derivative -> linear_step(1) -> model -> multipliers -> al_value, on the
    device (only the library's calls and torch arithmetic), against the same chain of restatements on the host."""
    import torch
    import __graft_entry__ as gent
    gent.build()
    import aligator_b200.gar as gar
    from oracle import gar_oracle, linesearch as ols, lq_assemble as olq
    B, N, nx, nu = 6, 8, 4, 2
    nc, nct, nc0 = nu, 0, nx
    mu, mu_dyn, preg = 0.05, 0.02, 1e-6
    rng = np.random.default_rng(7)
    model = _LqModel(rng, B, N, nx, nu)
    T = lambda a: torch.tensor(a, device="cuda", dtype=torch.float64)
    dm = model.on(T)
    it = dict(xs=rng.standard_normal((B, N + 1, nx)), us=0.8 * rng.standard_normal((B, N, nu)),
              lam0=rng.standard_normal((B, nc0)), lams=rng.standard_normal((B, N, nx)),
              vs=rng.standard_normal((B, N, nc)), vsT=np.zeros((B, nct)))
    prev_vs = rng.standard_normal((B, N, nc))
    lo, hi = -np.ones(nc), np.ones(nc)
    cJx, cJu = np.zeros((B, N, nc, nx)), np.broadcast_to(np.eye(nc, nu), (B, N, nc, nu)).copy()
    G0 = np.broadcast_to(np.eye(nx), (B, nx, nx)).copy()
    cm = lambda a: T(np.ascontiguousarray(np.swapaxes(a, -1, -2)))  # column-major device blocks
    D = dict(Jx=cm(model.A), Ju=cm(model.B), cJx=cm(cJx), cJu=cm(cJu), G0=cm(G0), Lxx=cm(model.Q),
             Luu=cm(model.R), Lxu=T(np.zeros((B, N, nx * nu))), Lxx_N=cm(model.Qn), lo=T(lo), hi=T(hi),
             prev_vs=T(prev_vs), prev_vsT=T(np.zeros((B, 0))), cval_N=T(np.zeros((B, 0))))
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    e = lambda *sh: torch.empty(*sh, device="cuda", dtype=torch.float64)
    z = lambda *sh: torch.zeros(*sh, device="cuda", dtype=torch.float64)
    def close(got, want, what, floor=0.0):
        """relative 1e-10; `floor` bounds the denominator below for arrays that vanish at the solution (a full step
        of a linear model leaves only round-off in the dynamics residual)"""
        got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
        err = np.linalg.norm((got - want).ravel()) / max(np.linalg.norm(want.ravel()), floor)
        if not err <= 1e-10:
            pytest.fail("%s: %.3e" % (what, err))

    def dev_multipliers(cur, ev):
        o = dict(slack=e(B, N, nx), lam0_plus=e(B, nc0), lams_plus=e(B, N, nx), vs_plus=e(B, N, nc),
                 vsT_plus=z(B, 0), shifted=e(B, N, nc), shifted_N=z(B, 0), Lv=e(B, N, nc), Lv_N=z(B, 0))
        inp = dict(xs=cur["xs"], lam0=cur["lam0"], lams=cur["lams"], vs=cur["vs"], vsT=cur["vsT"], xnext=ev["xnext"],
                   cval=ev["cval"], init_value=ev["init_value"], **{k: D[k] for k in ("prev_vs", "prev_vsT", "cval_N", "lo", "hi")})
        sc = s.multipliers(inp, o, mu, mu_dyn)
        return o, sc

    def host_multipliers(cur, ev):
        ms = [pin.compute_multipliers(list(cur["xs"][b]), [cur["lam0"][b]] + list(cur["lams"][b]),
                                      list(cur["vs"][b]) + [np.zeros(0)], list(prev_vs[b]) + [np.zeros(0)],
                                      ev["init_value"][b], list(ev["cval"][b]) + [np.zeros(0)], lo, hi, lo[:0], hi[:0],
                                      mu, mu_dyn, xnext=list(ev["xnext"][b])) for b in range(B)]
        return ms

    def check_multipliers(o, sc, ms, tag):
        assert np.all(sc[:, 1] == 1.0)
        close(o["slack"].cpu().numpy(), np.array([m["fs"][1:] for m in ms]), tag + " slack",
              floor=np.linalg.norm(np.array([m["fs"][0] for m in ms])) + 1.0)
        close(o["lams_plus"].cpu().numpy(), np.array([m["lams_plus"][1:] for m in ms]), tag + " lams_plus")
        close(o["lam0_plus"].cpu().numpy(), np.array([m["lams_plus"][0] for m in ms]), tag + " lam0_plus")
        close(o["vs_plus"].cpu().numpy(), np.array([m["vs_plus"][:N] for m in ms]), tag + " vs_plus")
        close(o["shifted"].cpu().numpy(), np.array([m["shifted"][:N] for m in ms]), tag + " shifted")
        close(o["Lv"].cpu().numpy(), np.array([m["Lvs"][:N] for m in ms]), tag + " Lv")
        close(sc[:, 0], np.array([m["prim_infeas"] for m in ms]), tag + " prim_infeas")

    def al_values(o, ev_dev, ms, ev_host, tag):
        plus = dict(lam0=o["lam0_plus"], lams=o["lams_plus"], vs=o["vs_plus"], vsT=o["vsT_plus"])
        got = s.al_value(plus, ev_dev["cost"], mu_dyn, mu)
        want = np.array([ols.al_value(ev_host["cost"][b], ms[b]["lams_plus"], ms[b]["vs_plus"], mu_dyn, mu, False)
                         for b in range(B)])
        close(got, want, tag + " al_value")
        return plus

    def lag(mult, ev):
        o = dict(Lx=e(B, N, nx), Lx_N=e(B, nx), Lu=e(B, N, nu), Lxs=e(B, N + 1, nx), Lus=e(B, N, nu))
        s.lagrangian_gradient(dict(lx=ev["lx"], lu=ev["lu"], lx_N=ev["lx_N"], Jx=D["Jx"], Ju=D["Ju"], cJx=D["cJx"],
                                   cJu=D["cJu"], G0=D["G0"], lam0=mult["lam0"], lams=mult["lams"], vs=mult["vs"],
                                   vsT=mult["vsT"]), o)
        return o

    def host_lag(b, lam_list, v_list, evh):
        return pin.lagrangian_gradient(list(evh["lx"][b]), list(evh["lu"][b]), evh["lx_N"][b], list(model.A[b]),
                                       list(model.B[b]), list(cJx[b]), list(cJu[b]), np.zeros((0, nx)), G0[b],
                                       lam_list, v_list)

    # ---- 1. multipliers and merit value at the iterate ----
    cur_d = {k: T(v) for k, v in it.items()}
    ev_d = dm.evaluate(cur_d["xs"], cur_d["us"])
    ev_h = model.evaluate(it["xs"], it["us"])
    o1, sc1 = dev_multipliers(cur_d, ev_d)
    ms1 = host_multipliers(it, ev_h)
    check_multipliers(o1, sc1, ms1, "iterate")
    plus1 = al_values(o1, ev_d, ms1, ev_h, "iterate")
    # ---- 2. Lagrangian gradient at the iterate's multipliers, criterion ----
    g1 = lag(cur_d, ev_d)
    hg = [host_lag(b, [it["lam0"][b]] + list(it["lams"][b]), list(it["vs"][b]) + [np.zeros(0)], ev_h) for b in range(B)]
    close(g1["Lxs"].cpu().numpy(), np.array([x for x, _ in hg]), "Lxs")
    close(g1["Lus"].cpu().numpy(), np.array([u for _, u in hg]), "Lus")
    crit = s.criterion(dict(Lxs=g1["Lxs"], Lus=g1["Lus"], init_value=ev_d["init_value"], slack=o1["slack"],
                            Lv=o1["Lv"], Lv_N=o1["Lv_N"]))
    crit_h = np.array([pin.criterion(hg[b][0], hg[b][1], ms1[b]["fs"], ms1[b]["Lvs"]) for b in range(B)])
    close(crit, crit_h, "criterion")
    # ---- 3. assemble + sweep ----
    s.assemble(dict(Jx=D["Jx"], Ju=D["Ju"], slack=o1["slack"], Lxx=D["Lxx"], Lxu=D["Lxu"], Luu=D["Luu"], Lx=g1["Lx"],
                    Lu=g1["Lu"], cJx=D["cJx"], cJu=D["cJu"], Lv=o1["Lv"], shifted=o1["shifted"], lo=D["lo"],
                    hi=D["hi"], Lxx_N=D["Lxx_N"], Lx_N=g1["Lx_N"], G0=D["G0"], g0=ev_d["init_value"]), preg, 1.0 / mu)
    srec = gar.stage_record_doubles(nx, nu, nc)
    packed = []
    for b in range(B):
        inp = dict(Jx=model.A[b], Ju=model.B[b], slack=np.array(ms1[b]["fs"][1:]), Lxx=model.Q[b],
                   Lxu=np.zeros((N, nx, nu)), Luu=model.R[b], Lx=np.array(hg[b][0][:N]), Lu=np.array(hg[b][1]),
                   cJx=cJx[b], cJu=cJu[b], Lv=np.array(ms1[b]["Lvs"][:N]), shifted=np.array(ms1[b]["shifted"][:N]),
                   lo=lo, hi=hi, Lxx_N=model.Qn[b], Lx_N=hg[b][0][N], G0=G0[b], g0=ev_h["init_value"][b],
                   preg=preg, mu_inv=1.0 / mu)
        packed.append(olq.pack(olq.assemble_problem(inp, N, nx, nu, nc, nct, nc0), N, nx, nu, nc, nct, srec))
    want = [np.stack([p[i] for p in packed]) for i in range(4)]
    for i in range(4):
        close(s.get_problem(i).reshape(want[i].shape), want[i], "assembled problem %d" % i)
    s.sweep(mu)
    assert np.all(s.status() == 0)
    bo = gar_oracle.BatchedOracle(nx, nu, nc, nct, nc0, N, B, *want)
    bo.sweep(mu, nthreads=1)
    ref = bo.get()
    step = dict(xs=s.get(gar.OUT_XS), us=s.get(gar.OUT_US), vs=s.get(gar.OUT_VS), lams=s.get(gar.OUT_LBDAS),
                lam0=s.get(gar.OUT_LBD0))
    for k, rk in (("xs", "xs"), ("us", "us"), ("vs", "vs"), ("lams", "lbdas"), ("lam0", "lbd0")):
        close(step[k], ref[rk], "step " + k)
    # ---- 4. gradient at the plus multipliers, directional derivative ----
    g2 = lag(plus1, ev_d)
    dphi = s.directional_derivative(g2["Lxs"], g2["Lus"])
    dphi_h = []
    for b in range(B):
        Lx2, Lu2 = host_lag(b, ms1[b]["lams_plus"], ms1[b]["vs_plus"], ev_h)
        dphi_h.append(ols.directional_derivative(Lx2, Lu2, list(ref["xs"][b]), list(ref["us"][b])))
    close(dphi, np.array(dphi_h), "directional derivative")
    # ---- 5. linear step alpha = 1, model, multipliers and merit value at the trial point ----
    trial = {k: torch.empty_like(v) for k, v in cur_d.items()}
    s.linear_step(1.0, cur_d, trial)
    tr_h = {}
    for b in range(B):
        tx, tu, tv, tl = ols.try_linear_step(list(it["xs"][b]), list(it["us"][b]), list(it["vs"][b]),
                                             [it["lam0"][b]] + list(it["lams"][b]), list(ref["xs"][b]),
                                             list(ref["us"][b]), list(ref["vs"][b]),
                                             [ref["lbd0"][b]] + list(ref["lbdas"][b]), 1.0)
        for k, v in (("xs", tx), ("us", tu), ("vs", tv), ("lam0", tl[:1]), ("lams", tl[1:])):
            tr_h.setdefault(k, []).append(np.array(v).reshape(np.shape(it[k][b])))
    tr_h = {k: np.array(v) for k, v in tr_h.items()}
    tr_h["vsT"] = np.zeros((B, 0))
    for k in ("xs", "us", "vs", "lam0", "lams"):
        close(trial[k].cpu().numpy(), tr_h[k], "trial " + k)
    ev2_d = dm.evaluate(trial["xs"], trial["us"])
    ev2_h = model.evaluate(tr_h["xs"], tr_h["us"])
    o2, sc2 = dev_multipliers(trial, ev2_d)
    ms2 = host_multipliers(tr_h, ev2_h)
    check_multipliers(o2, sc2, ms2, "trial")
    al_values(o2, ev2_d, ms2, ev2_h, "trial")
    s.close()
