"""Restatements of the theta derivatives of a parametric LQ solution (ab2_gar_theta_tangent / ab2_gar_theta_adjoint,
aligator_b200/csrc/lq_theta.cuh) on one instance's factors in the product's layouts (CudaRiccatiBatch.get, or
lq_cases.oracle_parametric): fb [N][nr][nx], fth [N][nr][nth], Vxx [N+1][nx][nx], Vxt [N+1][nx][nth],
kkt0fth [nx+nc0][nth], fbT [nct][nx].  Plain numpy: in fp64 they are the e_oracle side of the bar.  The
extended-precision side is theta_jacobian, built on hp_reference's backward pass and rollout.  The layouts and names
follow hp_reference (lbd0 for lam0, lbdas for lams)."""
import numpy as np

import hp_reference as hp

KEYS = ("xs", "us", "vs", "vsT", "lbd0", "lbdas")
FAMILIES = ("xs", "us", "vs", "lbd")


def theta_jacobian(p, mueq):
    """J = dz/dtheta of hp_reference.solve_parametric's solution, at its working precision: the reference's backward
    pass and initial system, then its rollout with the feed-forward vectors (ff, vx) dropped, started at kkt0fth and
    run at theta = I, so that column c is the rollout along the unit direction e_c.  -> dict of object arrays with
    theta last: xs [N+1][nx][nth], us [N][nu][nth], vs [N][nc][nth], vsT [nct][nth], lbd0 [nc0][nth],
    lbdas [N][nx][nth]."""
    N, nx, nc0 = p.horizon, p.stages[0].nx, p.nc0
    nth = p.stages[0].Gth.shape[0]
    st = [hp._mp_pknot(k) for k in p.stages]
    fac = hp._backward(st, hp.MP.mpf(float(mueq)))
    f0 = fac[0]
    G0 = hp.mpa(p.G0)
    M0 = np.block([[f0["Vxx"], G0.T], [G0, hp.zeros(nc0, nc0)]]) if nc0 else f0["Vxx"]
    kkt0fth = -hp.lu_solve(M0, np.concatenate([f0["Vxt"], hp.zeros(nc0, nth)]))
    lin = [dict(f, ff=hp.zeros(len(f["ff"]), 1), vx=hp.zeros(nx, 1)) for f in fac]
    xs, us, vs, lbdas = hp._rollout(st, lin, kkt0fth[:nx], hp.eye(nth))
    nu, nc = (p.stages[0].nu, p.stages[0].nc) if N else (0, 0)
    stack = lambda lst, *shape: np.stack(lst) if lst else hp.zeros(*shape)
    return dict(xs=np.stack(xs), us=stack(us, 0, nu, nth), vs=stack(vs[:N], 0, nc, nth), vsT=vs[N], lbd0=kkt0fth[nx:],
                lbdas=stack(lbdas, 0, nx, nth))


def tangent(f, d, nu, nc):
    """J d: the rollout of the theta terms from x_0 = F0_x d."""
    N, nx = f["fb"].shape[0], f["Vxx"].shape[-1]
    nk = nu + nc
    F0 = f["kkt0fth"]
    xs, us, vs, lbdas = [F0[:nx] @ d], [], [], []
    for t in range(N):
        y = f["fb"][t] @ xs[t] + f["fth"][t] @ d
        us.append(y[:nu]), vs.append(y[nu:nk]), xs.append(y[nk:])
        lbdas.append(f["Vxx"][t + 1] @ xs[t + 1] + f["Vxt"][t + 1] @ d)
    st = lambda lst, n: np.stack(lst) if lst else np.zeros((0, n))
    return dict(xs=np.stack(xs), us=st(us, nu), vs=st(vs, nc), vsT=f["fbT"] @ xs[N], lbd0=F0[nx:] @ d,
                lbdas=st(lbdas, nx))


def adjoint(f, z, nu, nc):
    """J^T zbar, zbar a dict with the keys of `tangent`'s result (missing = zero), by the transposed recursion."""
    N, nx = f["fb"].shape[0], f["Vxx"].shape[-1]
    F0 = f["kkt0fth"]
    nth = F0.shape[1]
    g = lambda k, *i: np.asarray(z[k][i]) if z.get(k) is not None else 0.0
    c = np.zeros(nx) + g("xs", N) + (f["fbT"].T @ z["vsT"] if z.get("vsT") is not None else 0.0)
    tb = np.zeros(nth)
    if N:
        c = c + f["Vxx"][N].T @ g("lbdas", N - 1)
        tb = f["Vxt"][N].T @ g("lbdas", N - 1)
    for t in range(N - 1, -1, -1):
        w = np.concatenate([np.broadcast_to(g("us", t), (nu,)), np.broadcast_to(g("vs", t), (nc,)), c])
        tb = tb + f["fth"][t].T @ w
        c = g("xs", t) + f["fb"][t].T @ w
        if t >= 1:
            tb = tb + f["Vxt"][t].T @ g("lbdas", t - 1)
            c = c + f["Vxx"][t].T @ g("lbdas", t - 1)
    lam0 = z.get("lbd0")
    return tb + F0[:nx].T @ c + (F0[nx:].T @ lam0 if lam0 is not None and F0.shape[0] > nx else 0.0)


def jacobian_apply(J, d):
    """J d on theta_jacobian's J (object arrays) for an fp64 direction d -> fp64 dict."""
    dm = hp.mpa(d)
    return {k: hp.to64(J[k] @ dm) for k in KEYS}


def jacobian_transpose_apply(J, z):
    """J^T zbar on theta_jacobian's J for fp64 cotangents z (dict of KEYS, missing = zero) -> fp64 [nth]."""
    tb = None
    for k in KEYS:
        if z.get(k) is None or J[k].size == 0:
            continue
        nth = J[k].shape[-1]
        part = hp.mpa(np.ravel(z[k])) @ J[k].reshape(-1, nth)
        tb = part if tb is None else tb + part
    return hp.to64(tb)


def snap(ref):
    """The extended-precision reference with its working-precision noise made exact zeros: entries below 1e-30 of
    the largest entry of any field (x_0 = F0_x d is exactly zero when G0 pins the initial state, and comes out ~1e-50
    of the other outputs, against which any fp64 result would have a relative error of 1e30)."""
    top = max(np.abs(v).max(initial=0.0) for v in ref.values())
    return {k: np.where(np.abs(v) <= 1e-30 * top, 0.0, v) for k, v in ref.items()}


def errors(got, ref, nu, nc, N):
    """Error families (xs, us, vs, lbd) of per-direction solution dicts [M][...] (M = directions x instances) against
    the fp64-rounded reference (snapped), at hp_reference's relative Frobenius measure per knot."""
    return hp.error_families(got, snap(ref), nu, nc, N, FAMILIES)


def theta_errors(got, ref):
    """Max over directions and instances of the relative error of theta_bar [M][nth]."""
    return {"thbar": max(hp._rel(a, b) for a, b in zip(got, ref))}
