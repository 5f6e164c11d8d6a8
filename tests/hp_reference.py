"""The sweep restated in extended precision (mpmath, 50 significant digits): the yardstick both fp64 implementations
are measured against.

Independent of the oracle: every saddle-point system -- each stage's [[Rhat, D^T], [D, -mu I]], the terminal knot's
nct rows, the initial [[Vxx_0, G0^T], [G0, 0]] -- is solved by plain Gaussian elimination with partial pivoting, so
nothing depends on Bunch-Kaufman pivot decisions.  The fp64 inputs are exact in this precision; what the sweep
computes from them is accurate to ~cond * 1e-50, far below anything fp64 can resolve.

`solve` returns the outputs in the product's layouts (fp64, rounded from the extended-precision values);
`error_families` measures an implementation against them, family by family.  `solve_parametric` is the recursion of
parametric problems (nth > 0) as the reference states it, `solve_legs` the parallel solver's legs and condensed system
on top of it (tests/test_hp_parametric.py pins both).

Derivatives of the solve, exact to far below fp64, without any derivative formula or with the closed forms evaluated in
extended precision: `tangent_problem` is the forward mode of every output of the sweep by central differences of the
recursion at 100 digits; `grad_solution` and `grad_factor` are the reverse modes of the solution and of the
factorisation, the restatements of tests/lq_adjoint_ref.py and tests/lq_factor_adjoint_ref.py evaluated on object
arrays.  `grad_errors`, `factor_errors` and `solution_errors` measure an implementation's derivatives against them."""
import mpmath
import numpy as np

import gen
import lq_adjoint_ref as aref

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


STAGE_BLOCKS = ("A", "B", "f", "Q", "S", "R", "q", "r", "C", "D", "d")
TERM_BLOCKS = ("Q", "q", "C", "d")


def _mp_knot(k):
    return {n: mpa(getattr(k, n)) for n in ("Q", "S", "R", "q", "r", "A", "B", "f", "C", "D", "d")}


def dims_of(p):
    """(nx, nu, nc, nct, nc0, N) of an LqrProblem, in the restatements' order."""
    N = p.horizon
    return (p.stages[0].nx, p.stages[0].nu if N else 0, p.stages[0].nc if N else 0, p.stages[N].nc, p.nc0, N)


def _record_blocks(rec, off, shapes):
    """{block: fp64 array} of one packed record (column-major matrix blocks)."""
    out = {}
    for n, shape in shapes.items():
        a, b = off[n]
        out[n] = np.asarray(rec[a:b], dtype=np.float64).reshape(shape[::-1]).T if len(shape) == 2 else \
            np.asarray(rec[a:b], dtype=np.float64)
    return out


def _displace(p, st, G0, g0, pdot, h):
    """The extended-precision data st (knot dicts), G0, g0 moved to p + h pdot.  pdot: one instance's tangent in the
    records' layouts, a dict with any of stage [N][srec], term [trec], G0 [nc0 * nx] (column-major), g0 [nc0] (a
    missing or None entry is zero).  Q, R and the terminal Q must move symmetrically."""
    nx, nu, nc, nct, nc0, N = dims_of(p)
    so, _ = aref.stage_offsets(nx, nu, nc)
    to, _ = aref.term_offsets(nx, nct)
    get = lambda k: None if pdot.get(k) is None else np.asarray(pdot[k], dtype=np.float64)
    move = lambda x, d: x + h * mpa(d)
    sd, td = get("stage"), get("term")
    for t in range(N + 1):
        k = p.stages[t]
        if t < N:
            if sd is None:
                continue
            d = _record_blocks(sd.reshape(N, -1)[t], so, {n: getattr(k, n).shape for n in STAGE_BLOCKS})
        else:
            if td is None:
                continue
            d = _record_blocks(td.ravel(), to, {n: getattr(k, n).shape for n in TERM_BLOCKS})
        for n, v in d.items():
            if n in ("Q", "R"):
                assert np.array_equal(v, v.T), "a tangent of %s must be symmetric" % n
            st[t][n] = move(st[t][n], v)
    if get("G0") is not None:
        G0 = move(G0, get("G0").reshape(nx, nc0).T)
    if get("g0") is not None:
        g0 = move(g0, get("g0").ravel())
    return st, G0, g0


def solve_problem(p, mueq, pdot=None, h=0):
    """One LqrProblem (uniform stage dims, terminal knot nu = 0) at penalty mueq -> dict of extended-precision
    outputs (object arrays) in the product's layouts.  With a data direction `pdot` (see _displace), the problem
    p + h pdot, its data formed exactly in the working precision."""
    N = p.horizon
    st = [_mp_knot(k) for k in p.stages]
    G0, g0 = mpa(p.G0), mpa(p.g0)
    if pdot is not None:
        st, G0, g0 = _displace(p, st, G0, g0, pdot, MP.mpf(h))
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


# ---------------------------------------------------------------------------------------------------------------------
# Parametric problems (nth > 0) and leg mode
# ---------------------------------------------------------------------------------------------------------------------
# The reference's recursion with theta, statement by statement.  With nc > 0 it is not the exact theta-derivative of
# the value function: Vxt leaves out Z^T Gv, vt leaves out Gv^T z and Vtt leaves out Gv^T Zth
# (riccati-kernel.hxx:298-310), and a terminal knot with nu = 0 ignores its Gv (:146-149).  The restatement follows
# the reference there too; where Gv = 0 the recursion is exact (tests/test_hp_parametric.py pins it).
PARAM_BLOCKS = ("Gx", "Gu", "Gv", "Gth", "gamma")


def _mp_pknot(k):
    d = _mp_knot(k)
    d.update({n: mpa(getattr(k, n)) for n in PARAM_BLOCKS})
    return d


def _kkt(m, Rh, mu):
    nc = m["C"].shape[0]
    return np.block([[Rh, m["D"].T], [m["D"], -mu * eye(nc)]]) if nc else Rh


def _terminal_solve(m, mu):
    """terminalSolve (riccati-kernel.hxx:131-193), both branches.  -> dict of the knot's factors: fb, ff, fth (rows
    [K; Z] only: a terminal knot has no closed loop), Vxx, vx and, with nth > 0, Vxt, Vtt, vt."""
    nu, nc, nth = m["R"].shape[0], m["C"].shape[0], m["Gth"].shape[0]
    if nu == 0:                                                                   # :146-149
        fb, ff, fth = m["C"] / mu, m["d"] / mu, zeros(nc, nth)
    else:                                                                         # :150-173
        rhs = np.concatenate([np.concatenate([m["S"].T, m["r"][:, None], m["Gu"]], axis=1),
                              np.concatenate([m["C"], m["d"][:, None], zeros(nc, nth)], axis=1)], axis=0)
        sol = -lu_solve(_kkt(m, m["R"], mu), rhs)
        fb, ff, fth = sol[:, :m["Q"].shape[0]], sol[:, m["Q"].shape[0]], sol[:, m["Q"].shape[0] + 1:]
    K, k, Z, z = fb[:nu], ff[:nu], fb[nu:], ff[nu:]
    o = dict(fb=fb, ff=ff, fth=fth, Vxx=m["Q"] + m["C"].T @ Z + m["S"] @ K, vx=m["q"] + m["C"].T @ z + m["S"] @ k)
    if nth:                                                                       # :185-192
        o.update(Vxt=m["Gx"] + K.T @ m["Gu"], Vtt=m["Gth"] + m["Gu"].T @ fth[:nu], vt=m["gamma"] + m["Gu"].T @ k)
    return o


def _stage_solve(m, n, mu):
    """stageKernelSolve (riccati-kernel.hxx:210-312) of knot m given the next knot's factors n; the theta columns
    are extra right-hand sides of the stage KKT system."""
    nx, nu, nc, nth = m["Q"].shape[0], m["R"].shape[0], m["C"].shape[0], m["Gth"].shape[0]
    V, v = n["Vxx"], n["vx"]
    vp = v + V @ m["f"]
    Qh = m["Q"] + m["A"].T @ V @ m["A"]
    Sh = m["S"] + m["A"].T @ V @ m["B"]
    Rh = m["R"] + m["B"].T @ V @ m["B"]
    qh = m["q"] + m["A"].T @ vp
    rh = m["r"] + m["B"].T @ vp
    top = [Sh.T, rh[:, None]] + ([m["Gu"] + m["B"].T @ n["Vxt"]] if nth else [])   # Guhat, :286-287
    bot = [m["C"], m["d"][:, None]] + ([m["Gv"]] if nth else [])
    sol = -lu_solve(_kkt(m, Rh, mu), np.concatenate([np.concatenate(top, axis=1), np.concatenate(bot, axis=1)]))
    KZ, kz = sol[:, :nx], sol[:, nx]
    K, k = KZ[:nu], kz[:nu]
    Ah, a = m["A"] + m["B"] @ K, m["f"] + m["B"] @ k
    o = dict(fb=np.concatenate([KZ, Ah], axis=0), ff=np.concatenate([kz, a]),
             Vxx=Qh + Sh @ K + m["C"].T @ KZ[nu:], vx=qh + Sh @ k + m["C"].T @ kz[nu:])
    if nth:
        KZth = sol[:, nx + 1:]
        Yth = m["B"] @ KZth[:nu]                                                  # :295
        o.update(fth=np.concatenate([KZth, Yth], axis=0),
                 vt=m["gamma"] + n["vt"] + m["Gu"].T @ k + n["Vxt"].T @ a,       # :298-301
                 Vxt=m["Gx"] + K.T @ m["Gu"] + Ah.T @ n["Vxt"],                   # :304-306
                 Vtt=m["Gth"] + n["Vtt"] + m["Gu"].T @ KZth[:nu] + n["Vxt"].T @ Yth)  # :308-310
    return o


def _backward(st, mu):
    """backwardImpl (riccati-kernel.hxx:105-129) over the knot dicts st: the last one by terminalSolve."""
    fac = [None] * len(st)
    fac[-1] = _terminal_solve(st[-1], mu)
    for t in range(len(st) - 2, -1, -1):
        fac[t] = _stage_solve(st[t], fac[t + 1], mu)
    return fac


def _rollout(st, fac, x0, theta):
    """forwardImpl (riccati-kernel.hxx:315-377) from x0 over the knots st; theta None or an object vector.  -> xs,
    us (one per knot with nu > 0), vs (one per knot), lbdas (the co-states of knots 1 .. n)."""
    xs, us, vs, lbdas = [x0], [], [], []
    n = len(st) - 1
    for t in range(n + 1):
        m, f, x = st[t], fac[t], xs[t]
        nu, nc = m["R"].shape[0], m["C"].shape[0]
        th = theta is not None and m["Gth"].shape[0] > 0
        if nu:
            us.append(f["fb"][:nu] @ x + f["ff"][:nu] + (f["fth"][:nu] @ theta if th else 0))
        vs.append(f["fb"][nu:nu + nc] @ x + f["ff"][nu:nu + nc] + (f["fth"][nu:nu + nc] @ theta if th else 0))
        if t == n:
            break
        xs.append(f["fb"][nu + nc:] @ x + f["ff"][nu + nc:] + (f["fth"][nu + nc:] @ theta if th else 0))
        g = fac[t + 1]
        lbdas.append(g["Vxx"] @ xs[t + 1] + g["vx"] + (g["Vxt"] @ theta if th else 0))
    return xs, us, vs, lbdas


def solve_parametric(p, mueq, theta=None):
    """One parametric LqrProblem (uniform stage dims, terminal nu = 0) at penalty mueq: the reference's backward pass
    with theta (riccati-kernel.hxx), the initial system with thGrad and thHess (proximal-riccati.hxx:39-60) and the
    rollout at theta (computeInitial, :196-207, then forwardImpl) -> dict of extended-precision outputs in the
    product's layouts: solve_problem's keys, and fth [N][nu+nc+nx][nth], Vxt [N+1][nx][nth], Vtt [N+1][nth][nth],
    vt [N+1][nth], kkt0 [nx+nc0], kkt0fth [nx+nc0][nth], thGrad [nth], thHess [nth][nth].  theta None: the
    theta-free rollout."""
    N, nx, nc0 = p.horizon, p.stages[0].nx, p.nc0
    nth = p.stages[0].Gth.shape[0]
    st = [_mp_pknot(k) for k in p.stages]
    mu = MP.mpf(float(mueq))
    fac = _backward(st, mu)
    G0, g0 = mpa(p.G0), mpa(p.g0)
    f0 = fac[0]
    M0 = np.block([[f0["Vxx"], G0.T], [G0, zeros(nc0, nc0)]]) if nc0 else f0["Vxx"]
    s0 = -lu_solve(M0, np.concatenate([np.concatenate([f0["vx"], g0])[:, None],
                                       np.concatenate([f0["Vxt"], zeros(nc0, nth)])], axis=1))   # :50-55
    kkt0, kkt0fth = s0[:, 0], s0[:, 1:]
    th = None if theta is None else mpa(theta)
    init = kkt0 + (kkt0fth @ th if th is not None else 0)                                           # :196-207
    xs, us, vs, lbdas = _rollout(st, fac, init[:nx], th)
    stack = lambda lst, *shape: np.stack(lst) if lst else zeros(*shape)
    nu, nc = (p.stages[0].nu, p.stages[0].nc) if N else (0, 0)
    return dict(fb=stack([f["fb"] for f in fac[:N]], 0, nu + nc + nx, nx),
                ff=stack([f["ff"] for f in fac[:N]], 0, nu + nc + nx),
                fth=stack([f["fth"] for f in fac[:N]], 0, nu + nc + nx, nth),
                Vxx=np.stack([f["Vxx"] for f in fac]), vx=np.stack([f["vx"] for f in fac]),
                Vxt=np.stack([f["Vxt"] for f in fac]), Vtt=np.stack([f["Vtt"] for f in fac]),
                vt=np.stack([f["vt"] for f in fac]), fbT=fac[N]["fb"], ffT=fac[N]["ff"],
                kkt0=kkt0, kkt0fth=kkt0fth,
                thGrad=f0["vt"] + f0["Vxt"].T @ kkt0[:nx], thHess=f0["Vtt"] + f0["Vxt"].T @ kkt0fth[:nx],  # :57-59
                xs=np.stack(xs), us=stack(us, 0, nu), vs=stack(vs[:N], 0, nc), vsT=vs[N], lbd0=init[nx:],
                lbdas=stack(lbdas, 0, nx))


def solve_parametric_batch(probs, mueq, thetas=None):
    """solve_parametric over a batch (thetas: None or [B][nth]) -> (fp64 outputs [B, ...], extended-precision dicts)."""
    mus = np.broadcast_to(np.asarray(mueq, dtype=np.float64), (len(probs),))
    hp = [solve_parametric(p, m, None if thetas is None else thetas[b]) for b, (p, m) in enumerate(zip(probs, mus))]
    return {k: np.stack([to64(h[k]) for h in hp]) for k in hp[0]}, hp


def get_work(N, i, T):
    """parallel-solver.hxx:23-28: the knots [beg, end) of leg i of T."""
    return i * (N + 1) // T, (i + 1) * (N + 1) // T


def solve_legs(p, mueq, T):
    """ParallelRiccatiSolver (parallel-solver.hxx:51-243) with T legs restated in extended precision: every knot of a
    leg but the last leg parameterised by nth = nx (addParameterization, :52-60), each leg's last knot configured as
    Gx = A^T, Gu = B^T, Gth = 0, gamma = f (:136-147) and solved by terminalSolve's nu > 0 branch, the condensed
    system as assembleCondensedSystem(0) builds it (:85-129) solved by Gaussian elimination (no refinement), and
    the legs' rollouts, each at theta = the next leg head's co-state (:209-243).  Also collapseFeedback as the
    reference states it (parallel-solver.hpp:41-51): K_0 - Kth_0 Vxt_0^T.

    -> dict of extended-precision outputs in the product's layouts (leg mode: nth = nx): solve_problem's keys, fth,
    Vxt, Vtt, vt (zero on the last leg's knots, which carry no parameters), `param` [N+1] (True on the knots that
    carry them) and `collapse` [nu][nx].  A leg's last knot has no closed loop: its Ahat, a and Yth rows are zero."""
    N, nx, nc0 = p.horizon, p.stages[0].nx, p.nc0
    nu, nc = p.stages[0].nu, p.stages[0].nc
    assert N > 0 and T >= 2
    mu = MP.mpf(float(mueq))
    legs = [get_work(N, i, T) for i in range(T)]
    st, fac = [None] * (N + 1), [None] * (N + 1)
    for i, (beg, end) in enumerate(legs):
        for t in range(beg, end):
            k = p.stages[t].copy()
            if i + 1 < T:
                k.addParameterization(nx)
                if t == end - 1:                                                  # configure_knot
                    k.Gx[...], k.Gu[...], k.Gth[...], k.gamma[...] = k.A.T, k.B.T, 0.0, k.f
            st[t] = _mp_pknot(k)
        fac[beg:end] = _backward(st[beg:end], mu)
    # the condensed system, blocks [lbd0 | x0 | theta_0 | x_h1 | theta_1 | ...]
    dims = [nc0, nx] + [nx] * (2 * (T - 1))
    off = np.concatenate([[0], np.cumsum(dims)])
    M, rhs = zeros(off[-1], off[-1]), zeros(off[-1])
    put = lambda i, j, blk: M.__setitem__((slice(off[i], off[i + 1]), slice(off[j], off[j + 1])), blk)
    put(0, 1, mpa(p.G0))
    put(1, 0, mpa(p.G0).T)
    put(1, 1, fac[0]["Vxx"])
    rhs[off[0]:off[1]], rhs[off[1]:off[2]] = -mpa(p.g0), -fac[0]["vx"]
    put(1, 2, fac[0]["Vxt"])
    put(2, 1, fac[0]["Vxt"].T)
    for i in range(T - 1):
        i0, i1 = legs[i]
        j = 2 * (i + 1)
        put(j, j, fac[i0]["Vtt"])
        put(j + 1, j + 1, fac[i1]["Vxx"])
        put(j, j + 1, -eye(nx))
        put(j + 1, j, -eye(nx))
        if i + 2 < T:
            put(j + 1, j + 2, fac[i1]["Vxt"])
            put(j + 2, j + 1, fac[i1]["Vxt"].T)
        rhs[off[j]:off[j + 1]], rhs[off[j + 1]:off[j + 2]] = -fac[i0]["vt"], -fac[i1]["vx"]
    sol = lu_solve(M, rhs[:, None])[:, 0]
    seg = lambda j: sol[off[j]:off[j + 1]]
    xs, us, vs, lbdas = [None] * (N + 1), [None] * N, [None] * (N + 1), [None] * N
    for i, (beg, end) in enumerate(legs):
        th = seg(2 * (i + 1)) if i + 1 < T else None
        x, u, v, lb = _rollout(st[beg:end], fac[beg:end], seg(2 * i + 1), th)
        xs[beg:end], vs[beg:end] = x, v
        us[beg:beg + len(u)] = u
        lbdas[beg:end - 1] = lb
        if i:
            lbdas[beg - 1] = seg(2 * i)
    nr = nu + nc + nx
    pad = lambda a, rows: np.concatenate([a, zeros(rows - a.shape[0], *a.shape[1:])]) if a.shape[0] < rows else a
    param = np.array([t < legs[-1][0] for t in range(N + 1)])
    par = lambda f, key, *shape: f[key] if key in f else zeros(*shape)
    fb0 = fac[0]["fb"]
    return dict(fb=np.stack([pad(f["fb"], nr) for f in fac[:N]]), ff=np.stack([pad(f["ff"], nr) for f in fac[:N]]),
                fth=np.stack([pad(par(f, "fth", nr, nx), nr) for f in fac[:N]]),
                Vxx=np.stack([f["Vxx"] for f in fac]), vx=np.stack([f["vx"] for f in fac]),
                Vxt=np.stack([par(f, "Vxt", nx, nx) for f in fac]), Vtt=np.stack([par(f, "Vtt", nx, nx) for f in fac]),
                vt=np.stack([par(f, "vt", nx) for f in fac]), fbT=fac[N]["fb"], ffT=fac[N]["ff"], param=param,
                xs=np.stack(xs), us=np.stack(us), vs=np.stack(vs[:N]).reshape(N, nc), vsT=vs[N], lbd0=seg(0),
                lbdas=np.stack(lbdas), collapse=fb0[:nu] - fac[0]["fth"][:nu] @ fac[0]["Vxt"].T)


def solve_legs_batch(probs, mueq, T):
    """solve_legs over a batch -> (fp64 outputs [B, ...], extended-precision dicts)."""
    mus = np.broadcast_to(np.asarray(mueq, dtype=np.float64), (len(probs),))
    hp = [solve_legs(p, m, T) for p, m in zip(probs, mus)]
    out = {k: np.stack([to64(h[k]) for h in hp]) for k in hp[0] if k != "param"}
    out["param"] = np.stack([h["param"] for h in hp])
    return out, hp


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
FAMILIES = ("K", "k", "Z", "z", "Ahat", "a", "Vxx", "vx", "xs", "us", "vs", "lbd",
            "Kth", "Zth", "Yth", "Vxt", "Vtt", "vt", "kkt0fth", "thGrad", "thHess", "collapse")
FLOOR = 64 * U   # below this two correct fp64 implementations are indistinguishable
FACTOR = 16      # how much worse than the oracle the kernel may be on the same inputs


def _rel(a, b):
    """Relative Frobenius error of a against b; the absolute error where b is exactly zero."""
    den = float(np.linalg.norm(np.ravel(b)))
    num = float(np.linalg.norm(np.ravel(a) - np.ravel(b)))
    return num / den if den > 0 else num


def _pieces(o, nu, nc, N):
    """family -> list of per-(instance, knot) blocks of output dict o (fp64, product layouts); families whose
    outputs o does not have are left out (an implementation that computes only the trajectory, or only the
    factorisation).  The parametric families: Kth, Zth, Yth (the row blocks of fth [b, t]), Vxt, Vtt, vt per knot,
    kkt0fth, thGrad, thHess per instance, each in the product's layout ([nx][nth] for Vxt); where o has `param`
    [B][N+1] (leg mode) only on the knots it marks.  collapse: collapse_feedback's first gain [b] ([nu][nx])."""
    traj = "xs" in o
    B = o["xs" if traj else "fb"].shape[0]
    P = {f: [] for f in FAMILIES}
    param = o.get("param")
    has = lambda b, t: param is None or param[b, t]
    for b in range(B):
        for t in range(N):
            if "fb" in o:
                fb, ff = o["fb"][b, t], o["ff"][b, t]
                P["K"].append(fb[:nu]); P["k"].append(ff[:nu])
                if nc:
                    P["Z"].append(fb[nu:nu + nc]); P["z"].append(ff[nu:nu + nc])
                if fb.shape[0] > nu + nc:
                    P["Ahat"].append(fb[nu + nc:]); P["a"].append(ff[nu + nc:])
            if "fth" in o and has(b, t):
                fth = o["fth"][b, t]
                P["Kth"].append(fth[:nu]); P["Yth"].append(fth[nu + nc:])
                if nc:
                    P["Zth"].append(fth[nu:nu + nc])
            if traj:
                if nc:
                    P["vs"].append(o["vs"][b, t])
                P["us"].append(o["us"][b, t]); P["lbd"].append(o["lbdas"][b, t])
        if (o["vsT"] if traj else o["fbT"]).shape[1]:
            if "fbT" in o:
                P["Z"].append(o["fbT"][b]); P["z"].append(o["ffT"][b])
            if traj:
                P["vs"].append(o["vsT"][b])
        if traj and o["lbd0"].shape[1]:
            P["lbd"].append(o["lbd0"][b])
        for t in range(N + 1):
            if "Vxx" in o:
                P["Vxx"].append(o["Vxx"][b, t]); P["vx"].append(o["vx"][b, t])
            if "Vxt" in o and has(b, t):
                P["Vxt"].append(o["Vxt"][b, t]); P["Vtt"].append(o["Vtt"][b, t]); P["vt"].append(o["vt"][b, t])
            if traj:
                P["xs"].append(o["xs"][b, t])
        for f in ("kkt0fth", "thGrad", "thHess", "collapse"):
            if f in o:
                P[f].append(o[f][b])
    return P


def error_families(got, ref, nu, nc, N, families=FAMILIES):
    """Max over instances and knots of the relative error of `got` against the fp64-rounded extended-precision
    outputs `ref`, per family (families without entries on either side are left out).  The knots that carry
    parameters are those `ref` marks (leg mode)."""
    if "param" in ref:
        got = dict(got, param=ref["param"])
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


def table(title, e_oracle, e_kernel, e_torch=None):
    """One row per family: the oracle's error, the kernel's and their ratio; with `e_torch`, the error of the fp64
    torch.autograd derivation beside them."""
    extra = lambda f: "" if e_torch is None else " %10.2e" % e_torch.get(f, float("nan"))
    rows = ["%s\n  %-8s %10s %10s %7s%s" % (title, "family", "e_oracle", "e_kernel", "ratio",
                                           "" if e_torch is None else " %10s" % "e_torch")]
    for f in e_kernel:
        ratio = e_kernel[f] / e_oracle[f] if e_oracle[f] > 0 else float("inf") if e_kernel[f] > 0 else 0.0
        rows.append("  %-8s %10.2e %10.2e %7.2f%s" % (f, e_oracle[f], e_kernel[f], ratio, extra(f)))
    return "\n".join(rows)


# ---------------------------------------------------------------------------------------------------------------------
# Derivatives
# ---------------------------------------------------------------------------------------------------------------------
TANGENT_DPS = 100      # working precision of the central differences
TANGENT_STEP = 1e-40   # rounding ~1e-100 cond / h, truncation ~h^2 cond^2: both far below 1e-30 for cond up to 1e11
SELF_CHECK = 1e-30     # the differences at h and at 2h agree to this, relative, output by output
NOISE = 1e-45          # the differences' rounding is ~1e-60 cond (cond <= 1e11): anything below this is zero
OUTPUT_KEYS = ("fb", "ff", "Vxx", "vx", "fbT", "ffT", "xs", "us", "vs", "vsT", "lbd0", "lbdas")


def _norm(a):
    return MP.sqrt(MP.fsum(v * v for v in np.ravel(a))) if np.size(a) else _ZERO


def tangent_problem(p, mueq, pdot, h=TANGENT_STEP):
    """The derivative of every output of the sweep of p along the data direction pdot (see _displace): central
    differences (y(p + h pdot) - y(p - h pdot)) / 2h of the recursion at TANGENT_DPS digits -> dict of object arrays
    keyed as solve_problem's outputs.  Checked against the differences at 2h: they agree to SELF_CHECK relative to the
    larger of the derivative and the output itself, output by output.  An entry below NOISE times that scale is the
    rounding of a derivative that is exactly zero (x_0 when G0 pins it, say) and is returned as exactly zero."""
    with MP.workdps(TANGENT_DPS):
        hh = MP.mpf(h)

        def central(step):
            plus, minus = solve_problem(p, mueq, pdot, step), solve_problem(p, mueq, pdot, -step)
            return {k: (plus[k] - minus[k]) / (2 * step) for k in OUTPUT_KEYS}, plus

        (d1, y), (d2, _) = central(hh), central(2 * hh)
        for k in OUTPUT_KEYS:
            scale = max(_norm(d1[k]), _norm(d2[k]), _norm(y[k]))
            assert _norm(d1[k] - d2[k]) <= SELF_CHECK * scale, (k, float(_norm(d1[k] - d2[k]) / scale))
            small = np.vectorize(lambda v: abs(v) <= NOISE * scale, otypes=[bool])(d1[k]) if d1[k].size else False
            d1[k] = np.where(small, _ZERO, d1[k])
    return d1


def tangents(probs, mueq, dots):
    """tangent_problem over a batch: dots is a dict of [B, ...] arrays in the records' layouts.  -> (fp64 dict [B, ...],
    list of extended-precision dicts)."""
    mus = np.broadcast_to(np.asarray(mueq, dtype=np.float64), (len(probs),))
    hp = [tangent_problem(p, m, {k: None if v is None else np.asarray(v)[b] for k, v in dots.items()})
          for b, (p, m) in enumerate(zip(probs, mus))]
    return {k: np.stack([to64(h[k]) for h in hp]) for k in hp[0]}, hp


def solution_dict(hps):
    """Per-instance extended-precision outputs -> the batched solution dict of tests/lq_adjoint_ref.py (object)."""
    st = lambda k: np.stack([h[k] for h in hps])
    return dict(xs=st("xs"), us=st("us"), vs=st("vs"), vsT=st("vsT"), lam0=st("lbd0"), lams=st("lbdas"))


def factor_dict(hps):
    """Per-instance extended-precision outputs -> the factorisation in the restatements' keys (object)."""
    st = lambda k: np.stack([h[k] for h in hps])
    return dict(ff=st("ff"), fb=st("fb"), vxx=st("Vxx"), vx=st("vx"), fft=st("ffT"), fbt=st("fbT"))


def records(probs):
    """The packed records (stage [B][N][srec] zero-padded, term, G0 column-major, g0) of a batch, fp64."""
    nx, nu, nc, nct, nc0, N = dims_of(probs[0])
    _, srec = aref.stage_offsets(nx, nu, nc)
    stage = np.zeros((len(probs), N, srec))
    for b, p in enumerate(probs):
        for t in range(N):
            r = gen.stage_record(p.stages[t])
            stage[b, t, :r.size] = r
    term = np.stack([gen.term_record(p.stages[N]) for p in probs])
    G0 = np.stack([np.asarray(p.G0, dtype=np.float64).ravel(order="F") for p in probs]).reshape(len(probs), nc0 * nx)
    g0 = np.stack([np.asarray(p.g0, dtype=np.float64) for p in probs]).reshape(len(probs), nc0)
    return stage, term, G0, g0


def _mus(mueq, B):
    return np.array([MP.mpf(float(m)) for m in np.broadcast_to(np.asarray(mueq, dtype=np.float64), (B,))],
                    dtype=object)


def grad_solution(probs, mueq, cot, hps=None):
    """Extended-precision gradient records of <cot, z(p)> (z the solution, cot in tests/lq_adjoint_ref.py's layouts,
    fp64): w = K^-1 cot is the extended-precision solve of the problem with its vectors replaced by -cot (exact), then
    lq_adjoint_ref.grad_records on object arrays.  hps: the problems' extended-precision outputs, if at hand."""
    import lq_resolve_ref as rref
    d6 = dims_of(probs[0])
    c = aref._full(cot, d6, len(probs))
    hj = dict(q=-c["xs"], r=-c["us"], d=-c["vs"], dN=-c["vsT"], g0=-c["lam0"], f=-c["lams"])
    if hps is None:
        _, hps = solve(probs, mueq)
    _, w = solve(rref.replaced_problems(probs, hj), mueq)
    return aref.grad_records(solution_dict(hps), solution_dict(w), d6)


def grad_factor(probs, mueq, cot, hps=None):
    """Extended-precision gradient records of <cot, factorisation> (cot in tests/lq_factor_adjoint_ref.py's keys and
    shapes, fp64): lq_factor_adjoint_ref.factor_adjoint on object arrays, fed with the extended-precision
    factorisation."""
    import lq_factor_adjoint_ref as fadj
    d6 = dims_of(probs[0])
    if hps is None:
        _, hps = solve(probs, mueq)
    stage, term, _, _ = records(probs)
    f = factor_dict(hps)
    return fadj.factor_adjoint(mpa(stage), mpa(term), f["ff"], f["fb"], f["vxx"], f["vx"], f["fft"], f["fbt"],
                               {k: None if v is None else mpa(v) for k, v in cot.items()}, d6, _mus(mueq, len(probs)),
                               solve=lu_solve)


def grads64(g):
    return {k: to64(v) for k, v in g.items()}


# error families of the derivatives: one per record block (gradients), per factor block (factor tangents), per
# trajectory family (solution tangents); each the worst per-(instance, knot) relative error
GRAD_FAMILIES = STAGE_BLOCKS + tuple("N" + n for n in TERM_BLOCKS) + ("G0", "g0")
FACTOR_FAMILIES = ("K", "k", "Z", "z", "Ahat", "a", "Vxx", "vx")
TRAJ_FAMILIES = ("xs", "us", "vs", "lbd")


def _grad_pieces(g, d6):
    nx, nu, nc, nct, nc0, N = d6
    so, _ = aref.stage_offsets(nx, nu, nc)
    to, _ = aref.term_offsets(nx, nct)
    tt = np.asarray(g["term"], dtype=np.float64)
    B = tt.shape[0]
    st, tt = np.asarray(g["stage"], dtype=np.float64).reshape(B, N, -1 if N else 0), tt.reshape(B, -1)
    G0, g0 = (np.asarray(g[k], dtype=np.float64).reshape(B, -1) for k in ("G0", "g0"))
    P = {f: [] for f in GRAD_FAMILIES}
    for b in range(B):
        for t in range(N):
            for n, (a, e) in so.items():
                P[n].append(st[b, t, a:e])
        for n, (a, e) in to.items():
            P["N" + n].append(tt[b, a:e])
        P["G0"].append(G0[b]); P["g0"].append(g0[b])
    return P


def grad_errors(got, ref, d6, families=GRAD_FAMILIES):
    """Per record block: the worst per-(instance, knot) relative error of the gradient records `got` against `ref`
    (the fp64-rounded extended-precision records); blocks of zero size are left out."""
    g, r = _grad_pieces(got, d6), _grad_pieces(ref, d6)
    return {f: max(_rel(a, b) for a, b in zip(g[f], r[f])) for f in families if r[f] and np.size(r[f][0])}


def factor_errors(got, ref, d6):
    """Per factor block (K .. vx): the worst per-(instance, knot) relative error of a factorisation (or its tangent,
    in the restatements' keys ff, fb, vxx, vx, fft, fbt) against `ref` in the same keys."""
    nx, nu, nc, nct, nc0, N = d6
    conv = lambda o: dict(fb=o["fb"], ff=o["ff"], Vxx=o["vxx"], vx=o["vx"], fbT=o["fbt"], ffT=o["fft"])
    return error_families(conv(got), conv(ref), nu, nc, N, FACTOR_FAMILIES)


def solution_errors(got, ref, d6):
    """Per trajectory family: the worst per-(instance, knot) relative error of a solution (or its tangent) in
    tests/lq_adjoint_ref.py's keys against `ref` in the same keys."""
    nx, nu, nc, nct, nc0, N = d6
    conv = lambda o: dict(xs=o["xs"], us=o["us"], vs=o["vs"], vsT=o["vsT"], lbd0=o["lam0"], lbdas=o["lams"])
    return error_families(conv(got), conv(ref), nu, nc, N, TRAJ_FAMILIES)


def solution_of(o):
    """hp_reference / oracle output keys -> tests/lq_adjoint_ref.py's solution keys."""
    return dict(xs=o["xs"], us=o["us"], vs=o["vs"], vsT=o["vsT"], lam0=o["lbd0"], lams=o["lbdas"])


def factor_of(o):
    """hp_reference / oracle output keys -> the restatements' factor keys."""
    return dict(ff=o["ff"], fb=o["fb"], vxx=o["Vxx"], vx=o["vx"], fft=o["ffT"], fbt=o["fbT"])


# ---------------------------------------------------------------------------------------------------------------------
# FDDP backward pass
# ---------------------------------------------------------------------------------------------------------------------
FDDP_FAMILIES = ("K", "k", "Vxx", "Vx", "Quuks")


def fddp_backward_pass(Jx, Ju, fs, Lxx, Lxu, Luu, Lx, Lu, Lxx_N, Lx_N, preg):
    """oracle/fddp.py (SolverFDDPTpl::backwardPass, solver-fddp.hxx:204-277) restated in extended precision, statement by
    statement, with the LLT solve of Quu replaced by plain Gaussian elimination.  Same arguments (one instance, fp64);
    returns the same keys as object arrays: K, k, Quuks (N entries), Vxx, Vx (N + 1)."""
    N = len(Jx)
    nx = np.shape(Lxx_N)[0]
    pr = MP.mpf(float(preg))
    Vxx, Vx = [None] * (N + 1), [None] * (N + 1)
    K, k, Quuks = [None] * N, [None] * N, [None] * N
    V = mpa(Lxx_N)
    for i in range(nx):
        V[i, i] += pr                                                             # :217
    Vxx[N] = V
    Vx[N] = mpa(Lx_N) + V @ mpa(fs[N])                                            # :216, :219-220
    for i in range(N - 1, -1, -1):
        J = np.hstack([mpa(Jx[i]), mpa(Ju[i])])                                   # :236
        nu = np.shape(Ju[i])[1]
        grad = np.concatenate([mpa(Lx[i]), mpa(Lu[i])]) + J.T @ Vx[i + 1]         # :239-240
        S = mpa(Lxu[i])
        hess = np.block([[mpa(Lxx[i]), S], [S.T, mpa(Luu[i])]]) + (J.T @ Vxx[i + 1]) @ J   # :243-245
        Qxx, Qxu, Quu = hess[:nx, :nx], hess[:nx, nx:], hess[nx:, nx:].copy()
        for j in range(nu):
            Quu[j, j] += pr                                                       # :246
        Qx, Qu = grad[:nx], grad[nx:]
        sol = lu_solve(Quu, np.column_stack([-Qu, -Qxu.T]))                       # :252-262
        k[i], K[i] = sol[:, 0], sol[:, 1:]
        Quuks[i] = Quu @ k[i]                                                     # :264
        vx = Qx + K[i].T @ Qu                                                     # :268-269
        v = Qxx + Qxu @ K[i]                                                      # :270-271
        for r in range(nx):                                                       # :272 selfadjointView<Lower>
            for c in range(r + 1, nx):
                v[r, c] = v[c, r]
        for r in range(nx):
            v[r, r] += pr                                                         # :273
        Vxx[i] = v
        Vx[i] = vx + v @ mpa(fs[i])                                               # :274-276
    return dict(K=K, k=k, Vxx=Vxx, Vx=Vx, Quuks=Quuks)


def fddp_errors(got, ref):
    """Per family of FDDP_FAMILIES: the worst relative error of any (instance, knot) block of ``got`` (lists over
    instances of dicts of per-knot fp64 blocks, Vxx compared on its lower triangle) against ``ref`` (the same of
    `fddp_backward_pass` outputs)."""
    out = {}
    for f in FDDP_FAMILIES:
        errs = []
        for g, r in zip(got, ref):
            for a, b in zip(g[f], r[f]):
                a, b = np.asarray(a, dtype=np.float64), to64(b)
                if f == "Vxx":
                    il = np.tril_indices(b.shape[0])
                    a, b = a[il], b[il]
                errs.append(_rel(a, b))
        out[f] = max(errs)
    return out
