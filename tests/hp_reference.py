"""The sweep restated in extended precision (mpmath, 50 significant digits): the yardstick both fp64 implementations
are measured against.

Independent of the oracle: every saddle-point system -- each stage's [[Rhat, D^T], [D, -mu I]], the terminal knot's
nct rows, the initial [[Vxx_0, G0^T], [G0, 0]] -- is solved by plain Gaussian elimination with partial pivoting, so
nothing depends on Bunch-Kaufman pivot decisions.  The fp64 inputs are exact in this precision; what the sweep
computes from them is accurate to ~cond * 1e-50, far below anything fp64 can resolve.

`solve` returns the outputs in the product's layouts (fp64, rounded from the extended-precision values);
`error_families` measures an implementation against them, family by family."""
import mpmath
import numpy as np

import gen

MP = mpmath.MPContext()
MP.dps = 50
U = 2.0 ** -53  # unit roundoff of fp64
_ZERO = MP.mpf(0)


def mpa(a):
    """fp64 array -> object array of extended-precision numbers (exact)."""
    a = np.asarray(a, dtype=np.float64)
    return np.array([MP.mpf(float(v)) for v in a.ravel()] or [_ZERO], dtype=object)[:a.size].reshape(a.shape)


def to64(a):
    return np.array([float(v) for v in np.ravel(a)], dtype=np.float64).reshape(np.shape(a))


def zeros(*shape):
    z = np.empty(shape, dtype=object)
    z.fill(_ZERO)
    return z


def eye(n):
    e = zeros(n, n)
    for i in range(n):
        e[i, i] = MP.mpf(1)
    return e


def lu_solve(M, Rhs):
    """Solve M X = Rhs (object arrays; Rhs 2-D) by Gaussian elimination with partial pivoting."""
    n = M.shape[0]
    A = np.concatenate([M, Rhs], axis=1).copy()
    for k in range(n):
        p = k + max(range(n - k), key=lambda i: abs(A[k + i, k]))
        if A[p, k] == 0:
            raise ZeroDivisionError("singular saddle-point system")
        if p != k:
            A[[k, p]] = A[[p, k]]
        for i in range(k + 1, n):
            if A[i, k] != 0:
                A[i, k:] = A[i, k:] - (A[i, k] / A[k, k]) * A[k, k:]
    X = A[:, n:]
    for k in range(n - 1, -1, -1):
        X[k] = (X[k] - A[k, k + 1:n] @ X[k + 1:]) / A[k, k] if k + 1 < n else X[k] / A[k, k]
    return X


def _mp_knot(k):
    return {n: mpa(getattr(k, n)) for n in ("Q", "S", "R", "q", "r", "A", "B", "f", "C", "D", "d")}


def solve_problem(p, mueq):
    """One LqrProblem (uniform stage dims, terminal knot nu = 0) at penalty mueq -> dict of extended-precision
    outputs (object arrays) in the product's layouts."""
    N = p.horizon
    st = [_mp_knot(k) for k in p.stages]
    nx, nu, nc = p.stages[0].nx, (p.stages[0].nu if N else 0), (p.stages[0].nc if N else 0)
    nct, nc0 = p.stages[N].nc, p.nc0
    mu = MP.mpf(float(mueq))
    T = st[N]
    Vxx, vx = [None] * (N + 1), [None] * (N + 1)
    # terminal knot: [Z; z] = [C; d] / mu
    fbT, ffT = T["C"] / mu, T["d"] / mu
    Vxx[N] = T["Q"] + T["C"].T @ fbT
    vx[N] = T["q"] + T["C"].T @ ffT
    fb, ff = [None] * N, [None] * N
    for t in range(N - 1, -1, -1):
        m = st[t]
        V, v = Vxx[t + 1], vx[t + 1]
        vp = v + V @ m["f"]
        Qh = m["Q"] + m["A"].T @ V @ m["A"]
        Sh = m["S"] + m["A"].T @ V @ m["B"]
        Rh = m["R"] + m["B"].T @ V @ m["B"]
        qh = m["q"] + m["A"].T @ vp
        rh = m["r"] + m["B"].T @ vp
        M = np.block([[Rh, m["D"].T], [m["D"], -mu * eye(nc)]]) if nc else Rh
        rhs = np.concatenate([np.concatenate([Sh.T, m["C"]], axis=0), np.concatenate([rh, m["d"]])[:, None]], axis=1)
        sol = -lu_solve(M, rhs)
        KZ, kz = sol[:, :nx], sol[:, nx]
        K, k = KZ[:nu], kz[:nu]
        Ah, a = m["A"] + m["B"] @ K, m["f"] + m["B"] @ k
        fb[t] = np.concatenate([KZ, Ah], axis=0)
        ff[t] = np.concatenate([kz, a])
        Vxx[t] = Qh + Sh @ K + m["C"].T @ KZ[nu:]
        vx[t] = qh + Sh @ k + m["C"].T @ kz[nu:]
    # initial saddle-point system [[Vxx_0, G0^T], [G0, 0]] [x0; lbd0] = -[vx_0; g0]
    G0, g0 = mpa(p.G0), mpa(p.g0)
    M0 = np.block([[Vxx[0], G0.T], [G0, zeros(nc0, nc0)]]) if nc0 else Vxx[0]
    s0 = -lu_solve(M0, np.concatenate([vx[0], g0])[:, None])[:, 0]
    xs, us, vs, lbdas = [s0[:nx]], [], [], []
    for t in range(N):
        x = xs[t]
        us.append(fb[t][:nu] @ x + ff[t][:nu])
        vs.append(fb[t][nu:nu + nc] @ x + ff[t][nu:nu + nc])
        xs.append(fb[t][nu + nc:] @ x + ff[t][nu + nc:])
        lbdas.append(Vxx[t + 1] @ xs[t + 1] + vx[t + 1])
    stack = lambda lst, *shape: np.stack(lst) if lst else zeros(*shape)
    return dict(fb=stack(fb, 0, nu + nc + nx, nx), ff=stack(ff, 0, nu + nc + nx), Vxx=np.stack(Vxx), vx=np.stack(vx),
                fbT=fbT, ffT=ffT, xs=np.stack(xs), us=stack(us, 0, nu), vs=stack(vs, 0, nc), vsT=fbT @ xs[N] + ffT,
                lbd0=s0[nx:], lbdas=stack(lbdas, 0, nx))


def solve(probs, mueq):
    """A batch of problems -> (fp64 outputs [B, ...] in the product's layouts, list of extended-precision dicts).
    mueq: a number or one value per instance."""
    mus = np.broadcast_to(np.asarray(mueq, dtype=np.float64), (len(probs),))
    hp = [solve_problem(p, m) for p, m in zip(probs, mus)]
    return {k: np.stack([to64(h[k]) for h in hp]) for k in hp[0]}, hp


def kkt_residual(p, mueq, h):
    """Relative residual of the whole-problem KKT system (gen.lqr_dense_kkt), evaluated in extended precision at the
    extended-precision solution h: ||K z + rhs||_inf / (||K||_inf ||z||_inf + ||rhs||_inf)."""
    K, rhs, offs = gen.lqr_dense_kkt(p, mueq)
    N, nc0 = p.horizon, p.nc0
    z = list(h["lbd0"])
    for t, m in enumerate(p.stages):
        z += list(h["xs"][t])
        if t < N:
            z += list(h["us"][t]) + list(h["vs"][t]) + list(h["lbdas"][t])
        else:
            z += list(h["vsT"])
    z = np.array(z, dtype=object)
    assert z.size == K.shape[0]
    res = max(abs(MP.fsum(MP.mpf(float(K[i, j])) * z[j] for j in np.nonzero(K[i])[0]) + MP.mpf(float(rhs[i])))
              for i in range(K.shape[0]))
    scale = float(np.abs(K).sum(axis=1).max()) * float(max(abs(v) for v in z)) + float(np.abs(rhs).max())
    return float(res) / scale


def stage_equation_residual(p, mueq, h):
    """Largest relative residual of the equations that define the gains, Vxx and vx at every knot: the stage KKT
    M [K k; Z z] = -[Shat^T rhat; C d], Vxx_t = Qhat + Shat K + C^T Z, and the terminal Z = C / mu."""
    N = p.horizon
    mu = MP.mpf(float(mueq))
    worst = 0.0
    rel = lambda r, s: float(max((abs(v) for v in np.ravel(r)), default=_ZERO)) / max(
        float(max((abs(v) for v in np.ravel(s)), default=_ZERO)), 1e-300)
    kt = _mp_knot(p.stages[N])
    worst = max(worst, rel(mu * h["fbT"] - kt["C"], kt["C"]))
    for t in range(N):
        m = _mp_knot(p.stages[t])
        nu, nc = m["R"].shape[0], m["C"].shape[0]
        V, v = h["Vxx"][t + 1], h["vx"][t + 1]
        vp = v + V @ m["f"]
        Qh, Sh = m["Q"] + m["A"].T @ V @ m["A"], m["S"] + m["A"].T @ V @ m["B"]
        Rh, rh = m["R"] + m["B"].T @ V @ m["B"], m["r"] + m["B"].T @ vp
        M = np.block([[Rh, m["D"].T], [m["D"], -mu * eye(nc)]]) if nc else Rh
        KZ = h["fb"][t][:nu + nc]
        kz = h["ff"][t][:nu + nc]
        rhs = np.concatenate([np.concatenate([Sh.T, m["C"]], axis=0), np.concatenate([rh, m["d"]])[:, None]], axis=1)
        worst = max(worst, rel(M @ np.concatenate([KZ, kz[:, None]], axis=1) + rhs, rhs))
        worst = max(worst, rel(Qh + Sh @ KZ[:nu] + m["C"].T @ KZ[nu:] - h["Vxx"][t], h["Vxx"][t]))
    return worst


# ---------------------------------------------------------------------------------------------------------------------
# Error families and the conditioning-aware tolerance
# ---------------------------------------------------------------------------------------------------------------------
FAMILIES = ("K", "k", "Z", "z", "Ahat", "a", "Vxx", "vx", "xs", "us", "vs", "lbd")
FLOOR = 64 * U   # below this two correct fp64 implementations are indistinguishable
FACTOR = 16      # how much worse than the oracle the kernel may be on the same inputs


def _rel(a, b):
    """Relative Frobenius error of a against b; the absolute error where b is exactly zero."""
    den = float(np.linalg.norm(np.ravel(b)))
    num = float(np.linalg.norm(np.ravel(a) - np.ravel(b)))
    return num / den if den > 0 else num


def _pieces(o, nu, nc, N):
    """family -> list of per-(instance, knot) blocks of output dict o (fp64, product layouts); families whose
    outputs o does not have are left out (an implementation that computes only the trajectory)."""
    B = o["xs"].shape[0]
    P = {f: [] for f in FAMILIES}
    for b in range(B):
        for t in range(N):
            if "fb" in o:
                fb, ff = o["fb"][b, t], o["ff"][b, t]
                P["K"].append(fb[:nu]); P["k"].append(ff[:nu])
                if nc:
                    P["Z"].append(fb[nu:nu + nc]); P["z"].append(ff[nu:nu + nc])
                if fb.shape[0] > nu + nc:
                    P["Ahat"].append(fb[nu + nc:]); P["a"].append(ff[nu + nc:])
            if nc:
                P["vs"].append(o["vs"][b, t])
            P["us"].append(o["us"][b, t]); P["lbd"].append(o["lbdas"][b, t])
        if o["vsT"].shape[1]:
            if "fbT" in o:
                P["Z"].append(o["fbT"][b]); P["z"].append(o["ffT"][b])
            P["vs"].append(o["vsT"][b])
        if o["lbd0"].shape[1]:
            P["lbd"].append(o["lbd0"][b])
        for t in range(N + 1):
            if "Vxx" in o:
                P["Vxx"].append(o["Vxx"][b, t]); P["vx"].append(o["vx"][b, t])
            P["xs"].append(o["xs"][b, t])
    return P


def error_families(got, ref, nu, nc, N, families=FAMILIES):
    """Max over instances and knots of the relative error of `got` against the fp64-rounded extended-precision
    outputs `ref`, per family (families without entries on either side are left out)."""
    g, r = _pieces(got, nu, nc, N), _pieces(ref, nu, nc, N)
    return {f: max(_rel(a, b) for a, b in zip(g[f], r[f])) for f in families
            if g[f] and len(g[f]) == len(r[f]) and sum(np.size(b) for b in r[f])}


def stack_solutions(per_instance):
    """list of per-instance output dicts -> one dict of [B, ...] arrays."""
    return {k: np.stack([np.asarray(o[k], dtype=np.float64) for o in per_instance]) for k in per_instance[0]}


def tolerance(e_oracle):
    return max(FACTOR * e_oracle, FLOOR)


def violations(e_kernel, e_oracle):
    """Families where the kernel is worse than the conditioning allows: e_kernel > max(16 e_oracle, 64 u)."""
    return {f: (e_kernel[f], e_oracle[f]) for f in e_kernel if not e_kernel[f] <= tolerance(e_oracle[f])}


def table(title, e_oracle, e_kernel):
    rows = ["%s\n  %-5s %10s %10s %7s" % (title, "family", "e_oracle", "e_kernel", "ratio")]
    for f in e_kernel:
        ratio = e_kernel[f] / e_oracle[f] if e_oracle[f] > 0 else float("inf") if e_kernel[f] > 0 else 0.0
        rows.append("  %-5s %10.2e %10.2e %7.2f" % (f, e_oracle[f], e_kernel[f], ratio))
    return "\n".join(rows)
