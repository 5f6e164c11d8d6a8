"""Input generators of the inner-iteration kernels (FDDP backward pass, LQ assembly, multipliers and Lagrangian
gradient) that several test modules and tools/compare_libs.py share."""
import numpy as np

INF = np.inf


def random_fddp(rng, B, N, nx, nu):
    w = lambda n, p: (lambda r: r @ r.T)(rng.standard_normal((n, p)))
    d = dict(Jx=np.zeros((B, N, nx, nx)), Ju=rng.uniform(-1, 1, (B, N, nx, nu)), fs=0.1 * rng.standard_normal((B, N + 1, nx)),
             Lxx=np.zeros((B, N, nx, nx)), Lxu=np.zeros((B, N, nx, nu)), Luu=np.zeros((B, N, nu, nu)),
             Lx=rng.uniform(-1, 1, (B, N, nx)), Lu=rng.uniform(-1, 1, (B, N, nu)), Lxx_N=np.zeros((B, nx, nx)),
             Lx_N=rng.uniform(-1, 1, (B, nx)))
    for b in range(B):
        for t in range(N):
            H = w(nx + nu, nx + nu + 1) / max(nx, nu)
            d["Lxx"][b, t], d["Lxu"][b, t], d["Luu"][b, t] = H[:nx, :nx], H[:nx, nx:], H[nx:, nx:]
            d["Jx"][b, t] = np.eye(nx) + 0.1 * rng.standard_normal((nx, nx)) / np.sqrt(nx)
        d["Lxx_N"][b] = w(nx, nx + 1) / nx
    return d


def random_inputs(rng, N, nx, nu, nc, nct, nc0, exact=True, init_hess=True):
    r = lambda *s: rng.standard_normal(s)
    sym = lambda a: 0.5 * (a + np.swapaxes(a, -1, -2))
    spd = lambda a: a @ np.swapaxes(a, -1, -2) / a.shape[-1] + np.eye(a.shape[-1])  # well-posed sweeps
    inp = dict(Jx=np.eye(nx) + 0.1 * r(N, nx, nx), Ju=r(N, nx, nu), slack=r(N, nx), Lxx=spd(r(N, nx, nx)),
               Lxu=0.1 * r(N, nx, nu), Luu=spd(r(N, nu, nu)), Lx=r(N, nx), Lu=r(N, nu), Lxx_N=spd(r(nx, nx)),
               Lx_N=r(nx), preg=1e-3 * (1 + rng.random()), mu_inv=10.0 ** rng.integers(1, 4))
    if exact:
        inp.update(Hxx=0.01 * sym(r(N, nx, nx)), Hxu=0.01 * r(N, nx, nu), Huu=0.01 * sym(r(N, nu, nu)))
    if nc:
        # mixed product set: equality rows (always active), negative-orthant rows, box rows
        kinds = rng.integers(0, 3, nc)
        lo = np.where(kinds == 0, np.inf, np.where(kinds == 1, -np.inf, -0.5))
        hi = np.where(kinds == 0, np.inf, np.where(kinds == 1, 0.0, 0.5))
        inp.update(cJx=r(N, nc, nx), cJu=r(N, nc, nu), Lv=r(N, nc), shifted=r(N, nc), lo=lo, hi=hi)
    if nct:
        inp.update(cJx_N=r(nct, nx), Lv_N=r(nct), shifted_N=r(nct), loN=np.full(nct, -np.inf), hiN=np.zeros(nct))
    if nc0:
        inp.update(G0=r(nc0, nx), g0=r(nc0))
    if init_hess:
        inp["Hxx0"] = 0.01 * sym(r(nx, nx))
    return inp


# ---------------------------------------------------------------------------------------------------------------
# CPU: the restatement
# ---------------------------------------------------------------------------------------------------------------
def hand_case():
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


def hand_gradient_inputs():
    return dict(lx=[np.array([0.5, 0.5])], lu=[np.array([1.0])], lx_N=np.array([1.0, 1.0]),
                Jx=[np.array([[1.0, 2.0], [3.0, 4.0]])], Ju=[np.array([[1.0], [5.0]])],
                cJx=[np.array([[1.0, 0.0], [0.0, 1.0], [1.0, 1.0]])], cJu=[np.array([[0.0], [1.0], [2.0]])],
                cJx_N=np.array([[2.0, -1.0]]), G0=np.array([[1.0, 0.0], [0.0, 2.0]]))


# ---------------------------------------------------------------------------------------------------------------------
# FDDP: the extended-precision backward pass
# ---------------------------------------------------------------------------------------------------------------------
def fddp_case(name, rng, B, N, nx, nu):
    """test_fddp's random problems, and the variants of the level-2 FDDP tests: 'singular' (the last control direction
    scaled by 1e-5 in Ju, Lxu, Luu: Quu's smallest eigenvalue ~1e-10, preg 1e-10), 'defects' (fs ~ 1e3)."""
    d = random_fddp(rng, B, N, nx, nu)
    preg = 1e-4
    if name == "singular":
        s = np.ones(nu)
        s[-1] = 1e-5
        d["Ju"] = d["Ju"] * s
        d["Lxu"] = d["Lxu"] * s
        d["Luu"] = d["Luu"] * s[:, None] * s
        preg = 1e-10
    elif name == "defects":
        d["fs"] = 1e3 * rng.standard_normal(d["fs"].shape)
    return d, preg


def fddp_args(d, b):
    return ([list(d[k][b]) for k in ("Jx", "Ju")] + [list(d["fs"][b])]
            + [list(d[k][b]) for k in ("Lxx", "Lxu", "Luu", "Lx", "Lu")] + [d["Lxx_N"][b], d["Lx_N"][b]])
