"""Element-wise exact references of the kernels around the sweep in the device-resident inner iteration: the LQ assembly
(DESIGN 2c), the line-search consumers (2e) and the multipliers / Lagrangian gradient / criterion (2g).

Each reference takes one instance's fp64 inputs and returns, per output element, what the kernel must produce:
  * a float: the element must be that double bit for bit (copies, zeroed rows, the normal-cone projection, one-rounding
    operations such as a linear-step element or a difference);
  * a `Bound(exact, T, m)`: the element is a sum of m products whose exact value is `exact` (a Fraction) and whose terms'
    magnitudes add up to T; any fp64 evaluation lies within gamma_{m+1} T of it (tests/exact_bounds.py).
Each follows the computation as the reference library writes it (the solver-proxddp.hxx / lagrangian.hpp /
merit-function.hxx lines the kernels cite), not a simplified equivalent: e.g. a constraint correction is P^T lv minus
Ptilde^T lv, two full sums and then a difference, so T counts both sums.  Where a decision depends on an earlier rounded
output (the projection on `shifted`, lams_plus on the slack), the reference takes the device's own value of it, which is
checked separately.

Matrices are given in math layout [rows, cols] (the device's blocks are column-major); per-knot arrays lead with the
knot index, as the device's per-instance arrays do."""
from fractions import Fraction

import numpy as np

from exact_bounds import bound, correctly_rounded, exact_sum, excess, same_bits, within



class Bound:
    """An element that is a sum of m terms with exact value ``exact`` and sum of magnitudes ``T`` (Fractions).  Not a
    tuple, so that numpy keeps it as one element of an object array."""
    __slots__ = ("exact", "T", "m")

    def __init__(self, exact, T, m):
        self.exact, self.T, self.m = exact, T, m

    def __iter__(self):
        return iter((self.exact, self.T, self.m))

    def __repr__(self):
        return "Bound(%.17g, T=%.3g, m=%d)" % (float(self.exact), float(self.T), self.m)


INF = float("inf")


def _bound(terms, m=None):
    e, T, n = exact_sum(terms)
    return Bound(e, T, n if m is None else m)


def _f(x):
    return float(x)


def obj(shape):
    return np.empty(shape, dtype=object)


def failures(got, want):
    """Indices (as tuples) where the device array ``got`` misses ``want`` (an object array of floats and Bounds, or a
    float array meaning bit for bit), with the element and what was expected."""
    got = np.asarray(got, dtype=np.float64)
    assert got.shape == np.shape(want), (got.shape, np.shape(want))
    if isinstance(want, np.ndarray) and want.dtype != object:
        bad = ~same_bits(got, want)
        return [(i, got[i], want[i]) for i in zip(*np.nonzero(bad))]
    out = []
    for i in np.ndindex(got.shape):
        w = want[i]
        ok = within(got[i], w.exact, w.T, w.m) if isinstance(w, Bound) else bool(same_bits(got[i], w))
        if not ok:
            out.append((i, float(got[i]), w if not isinstance(w, Bound) else (float(w.exact), excess(got[i], *w))))
    return out


def worst_excess(got, want):
    """max |got - exact| / (gamma T) over the Bound entries (<= 1 passes): the margin, for the printed tables."""
    r = [excess(g, *w) for g, w in zip(np.ravel(got), np.ravel(want)) if isinstance(w, Bound)]
    return max(r) if r else 0.0


# ---------------------------------------------------------------------------------------------------------------------
# Normal-cone projection (equality-constraint.hpp:37-40, box-constraint.hpp:27-37)
# ---------------------------------------------------------------------------------------------------------------------
def normal_cone(z, lo, hi):
    """One row, as the reference evaluates it: z on an equality row (lo = +inf), else z - max(min(z, hi), lo) with
    std::min(z, hi) = (hi < z ? hi : z) and std::max(c, lo) = (c < lo ? lo : c) -- the comparisons Eigen's
    cwiseMin(hi).cwiseMax(lo) makes, which decide the sign of a zero and what a NaN gives."""
    z, lo, hi = float(z), float(lo), float(hi)
    if lo == INF:
        return z
    c = hi if hi < z else z
    c = lo if c < lo else c
    return z - c


def active(z, lo, hi):
    """computeActiveSet of the product set (equality-constraint.hpp:52-55, negative-orthant.hpp:30-33,
    box-constraint.hpp:39-43): the row is active iff z > hi or z < lo."""
    return bool(z > hi or z < lo)


# ---------------------------------------------------------------------------------------------------------------------
# computeMultipliers (solver-proxddp.hxx:220-318)
# ---------------------------------------------------------------------------------------------------------------------
def multipliers(inp, got, lo, hi, loN, hiN, mu, mu_dyn):
    """One instance.  ``inp``: xs [N+1, nx], lam0, lams [N, nx], vs [N, nc], vsT, prev_vs, prev_vsT, init_value, cval,
    cval_N and one of xnext / fs [N, nx]; ``got``: the device's outputs of this instance (its slack, shifted and
    shifted_N enter).  Returns {output: want} and 'prim': the interval [lo, hi] (Fractions) the primal infeasibility
    must lie in.  Inputs and outputs must be finite (an instance whose flag is 0 is checked by the flag alone)."""
    mu, mu_dyn = float(mu), float(mu_dyn)
    mu_inv = 1.0 / mu                                                              # mu_inv() = 1 / mu()
    inv_mu, inv_mu_dyn = 1 / Fraction(mu), 1 / Fraction(mu_dyn)
    N, nx = inp["lams"].shape
    w = {}
    if inp.get("fs") is not None:                                                  # the caller's fs: copied
        w["slack"] = np.array(inp["fs"], dtype=np.float64)
    else:                                                                          # difference(x_{t+1}, xnext): one rounding
        w["slack"] = np.array([[correctly_rounded(Fraction(_f(a)) - Fraction(_f(b))) for a, b in zip(xn, x)]
                               for xn, x in zip(inp["xnext"], inp["xs"][1:])]).reshape(N, nx)
    # lams_plus[0] = lams[0] + fs[0] / mu(), lams_plus[t+1] = lams[t+1] + fs[t+1] / mu_dyn()   (:247, :264)
    w["lam0_plus"] = np.array([_bound([(_f(l),), (_f(f), inv_mu)]) for l, f in zip(inp["lam0"], inp["init_value"])] or [],
                              dtype=object)
    lp = obj((N, nx))
    for i in np.ndindex(N, nx):
        lp[i] = _bound([(_f(inp["lams"][i]),), (_f(got["slack"][i]), inv_mu_dyn)])
    w["lams_plus"] = lp
    prim = [(Fraction(abs(_f(f))),) * 2 for f in list(np.ravel(inp["init_value"])) + list(np.ravel(got["slack"]))]

    def rows(cval, prev, vs, shifted, lo_, hi_):
        n = len(cval)
        sh, lv, vp = obj(n), obj(n), np.empty(n)
        for i in range(n):
            sh[i] = _bound([(_f(cval[i]),), (mu, _f(prev[i]))])                    # cval + mu vs_prev   (:277)
            nc = normal_cone(shifted[i], lo_[i], hi_[i])                            # on the device's shifted   (:278)
            lv[i] = _bound([(nc,), (-mu, _f(vs[i]))])                               # NC - mu vs   (:281-282)
            vp[i] = mu_inv * nc                                                     # mu_inv NC: one rounding   (:283)
            e = _bound([(mu, vp[i]), (-mu, _f(prev[i]))])                           # mu (vs_plus - vs_prev)   (:286)
            g = bound(e.T, e.m)
            prim.append((max(abs(e.exact) - g, Fraction(0)), abs(e.exact) + g))
        return sh, lv, vp

    nc = inp["cval"].shape[1] if inp["cval"].ndim == 2 else 0
    sh, lv, vp = rows(np.ravel(inp["cval"]), np.ravel(inp["prev_vs"]), np.ravel(inp["vs"]), np.ravel(got["shifted"]),
                      np.tile(lo, N), np.tile(hi, N))
    w["shifted"], w["Lv"], w["vs_plus"] = sh.reshape(N, nc), lv.reshape(N, nc), vp.reshape(N, nc)
    w["shifted_N"], w["Lv_N"], w["vsT_plus"] = rows(inp["cval_N"], inp["prev_vsT"], inp["vsT"], got["shifted_N"], loN, hiN)
    w["prim"] = (max([p[0] for p in prim] + [Fraction(0)]), max([p[1] for p in prim] + [Fraction(0)]))  # (:315-316)
    return w


def flag(got):
    """RET_FALSE_IF_NAN's verdict on the device's own lams_plus (both) and Lvs (both): 1.0 when all are finite."""
    return 1.0 if all(np.all(np.isfinite(got[k])) for k in ("lam0_plus", "lams_plus", "Lv", "Lv_N")) else 0.0


# ---------------------------------------------------------------------------------------------------------------------
# LagrangianDerivatives::compute (lagrangian.hpp:29-92) + innerLoop's Lxs[0].setZero() (solver-proxddp.hxx:592-594)
# ---------------------------------------------------------------------------------------------------------------------
def lagrangian_gradient(g, force_initial_condition=False, knots=None):
    """One instance.  ``g``: lx [N, nx], lu [N, nu], lx_N, Jx [N, nx, nx], Ju [N, nx, nu], cJx [N, nc, nx],
    cJu [N, nc, nu], cJx_N [nct, nx], G0 [nc0, nx], lam0, lams [N, nx], vs [N, nc], vsT.  Returns (Lxs [N+1, nx],
    Lus [N, nu]) as object arrays; rows of knots not in ``knots`` (default: all) are None.
        Lxs[t] = lx_t + Jx_t^T lam_{t+1} + cJx_t^T v_t (+ G0^T lam0 at t = 0) (- lam_t at t >= 1)
        Lus[t] = lu_t + Ju_t^T lam_{t+1} + cJu_t^T v_t
    (the terminal knot: lx_N + cJx_N^T v_N - lam_N, with G0^T lam0 when N = 0)."""
    N, nx = g["lams"].shape
    nu = g["lu"].shape[1]
    Lxs, Lus = obj((N + 1, nx)), obj((N, nu))
    fl = lambda a: [float(v) for v in np.ravel(a)]
    for t in (range(N + 1) if knots is None else knots):
        term = t == N
        Jx, cJx = (None, g["cJx_N"]) if term else (g["Jx"][t], g["cJx"][t])
        y2 = g["vsT"] if term else g["vs"][t]
        for c in range(nx):
            if t == 0 and force_initial_condition:
                Lxs[t, c] = 0.0
                continue
            terms = [(float(g["lx_N"][c] if term else g["lx"][t, c]),)]                    # :60, :84
            if not term:
                terms += [(a, b) for a, b in zip(fl(Jx[:, c]), fl(g["lams"][t]))]             # :63
            terms += [(a, b) for a, b in zip(fl(cJx[:, c]), fl(y2))]                         # :70, :89
            if t == 0:
                terms += [(a, b) for a, b in zip(fl(g["G0"][:, c]), fl(g["lam0"]))]          # :52-53
            else:
                terms.append((-1.0, float(g["lams"][t - 1, c])))                             # :75
            Lxs[t, c] = _bound(terms)
        if not term:
            for c in range(nu):
                terms = [(float(g["lu"][t, c]),)]                                            # :61
                terms += [(a, b) for a, b in zip(fl(g["Ju"][t][:, c]), fl(g["lams"][t]))]    # :64
                terms += [(a, b) for a, b in zip(fl(g["cJu"][t][:, c]), fl(g["vs"][t]))]     # :71
                Lus[t, c] = _bound(terms)
    return Lxs, Lus


# ---------------------------------------------------------------------------------------------------------------------
# computeCriterion (solver-proxddp.hxx:703-732): maxima of the device's own arrays, exact
# ---------------------------------------------------------------------------------------------------------------------
def criterion(Lxs, Lus, init_value, slack, Lv, Lv_N):
    """One instance -> (inner_criterion, dual_infeas).  Stage i's dynamics residual is fs[i]: init_value for stage 0,
    slack knots 0 .. N-2 for stages 1 .. N-1 (the last slack is not counted)."""
    N = Lus.shape[0]
    m = lambda a: float(np.max(np.abs(a))) if np.size(a) else 0.0
    dual = max(m(Lxs), m(Lus))
    other = max(m(init_value) if N else 0.0, m(slack[:max(N - 1, 0)]), m(Lv), m(Lv_N))
    return max(dual, other), dual


# ---------------------------------------------------------------------------------------------------------------------
# updateLQSubproblem + computeProjectedJacobians (solver-proxddp.hxx:25-69, 734-805)
# ---------------------------------------------------------------------------------------------------------------------
def _corr(P, Lv, shifted, lo, hi, mu_inv):
    """Column j of P^T lv - Ptilde^T lv, lv = Lv mu_inv (one rounding per row, :46 / :63), Ptilde = P with the inactive
    rows zeroed: both sums over all rows, then the difference (:47-52, :64-68).  -> per column the terms with their
    signs and the count the rounding bound needs (two sums of nrows terms, the difference, the addition to q)."""
    nrows, ncols = P.shape
    lv = [float(np.float64(a) * np.float64(mu_inv)) for a in Lv]
    act = [active(shifted[i], lo[i], hi[i]) for i in range(nrows)]
    cols = []
    for j in range(ncols):
        full = [(float(P[i, j]), lv[i]) for i in range(nrows)]
        proj = [(-float(P[i, j]), lv[i]) for i in range(nrows) if act[i]]
        cols.append(full + proj)
    return cols, 2 * nrows + 2


def _zero_inactive(P, shifted, lo, hi):
    out = np.array(P, dtype=np.float64, copy=True)
    for i in range(P.shape[0]):
        if not active(shifted[i], lo[i], hi[i]):
            out[i, :] = 0.0                                                                   # +0.0
    return out


def assemble(inp, N, nx, nu, nc, nct, nc0, preg, mu_inv, knots=None):
    """One instance.  ``inp``: the ab2_lq_inputs arrays of this instance in math layout (Hxx, Hxu, Huu, Hxx0 optional;
    lo, hi, loN, hiN shared).  Returns {'stages': {t: {block: want}}, 'term': {block: want}, 'G0', 'g0'} for the
    knots in ``knots`` (default: all)."""
    preg, mu_inv = float(preg), float(mu_inv)
    stages = {}
    H = lambda k, t: inp.get(k)[t] if inp.get(k) is not None else None
    for t in (range(N) if knots is None else knots):
        k = {"A": np.array(inp["Jx"][t], dtype=np.float64), "B": np.array(inp["Ju"][t], dtype=np.float64),
             "f": np.array(inp["slack"][t], dtype=np.float64)}                                 # :755-757
        for name, L, Hs, n1, n2, diag in (("Q", "Lxx", "Hxx", nx, nx, True), ("S", "Lxu", "Hxu", nx, nu, False),
                                           ("R", "Luu", "Huu", nu, nu, True)):
            b = obj((n1, n2))
            for i, j in np.ndindex(n1, n2):
                terms = [(float(inp[L][t][i, j]),)]                                           # :759-761
                if diag and i == j:
                    terms.append((preg,))                                                     # :767-768
                if H(Hs, t) is not None:
                    terms.append((float(H(Hs, t)[i, j]),))                                    # :770-774
                if name == "Q" and t == 0 and inp.get("Hxx0") is not None:
                    terms.append((float(inp["Hxx0"][i, j]),))                                 # :803-804
                b[i, j] = _bound(terms)
            k[name] = b
        if nc:
            cx, m = _corr(inp["cJx"][t], inp["Lv"][t], inp["shifted"][t], inp["lo"], inp["hi"], mu_inv)
            cu, _ = _corr(inp["cJu"][t], inp["Lv"][t], inp["shifted"][t], inp["lo"], inp["hi"], mu_inv)
        else:
            cx, cu, m = [[] for _ in range(nx)], [[] for _ in range(nu)], 1
        k["q"] = np.array([_bound([(float(inp["Lx"][t][j]),)] + cx[j], m) for j in range(nx)], dtype=object)   # :764, :782
        k["r"] = np.array([_bound([(float(inp["Lu"][t][j]),)] + cu[j], m) for j in range(nu)], dtype=object)   # :765, :783
        if nc:
            k["C"] = _zero_inactive(inp["cJx"][t], inp["shifted"][t], inp["lo"], inp["hi"])    # :778
            k["D"] = _zero_inactive(inp["cJu"][t], inp["shifted"][t], inp["lo"], inp["hi"])
            k["d"] = np.array(inp["Lv"][t], dtype=np.float64)                                  # :780
        else:
            k["C"], k["D"], k["d"] = np.zeros((0, nx)), np.zeros((0, nu)), np.zeros(0)
        stages[t] = k
    term = {}
    Q = obj((nx, nx))
    for i, j in np.ndindex(nx, nx):
        terms = [(float(inp["Lxx_N"][i, j]),)] + ([(preg,)] if i == j else [])                 # :787-789
        if N == 0 and inp.get("Hxx0") is not None:
            terms.append((float(inp["Hxx0"][i, j]),))
        Q[i, j] = _bound(terms)
    term["Q"] = Q
    if nct:
        cx, m = _corr(inp["cJx_N"], inp["Lv_N"], inp["shifted_N"], inp["loN"], inp["hiN"], mu_inv)
        term["C"] = _zero_inactive(inp["cJx_N"], inp["shifted_N"], inp["loN"], inp["hiN"])    # :791
        term["d"] = np.array(inp["Lv_N"], dtype=np.float64)                                    # :792
    else:
        cx, m = [[] for _ in range(nx)], 1
        term["C"], term["d"] = np.zeros((0, nx)), np.zeros(0)
    term["q"] = np.array([_bound([(float(inp["Lx_N"][j]),)] + cx[j], m) for j in range(nx)], dtype=object)   # :790, :794
    G0 = np.array(inp["G0"], dtype=np.float64) if nc0 else np.zeros((0, nx))                   # :799-800
    g0 = np.array(inp["g0"], dtype=np.float64) if nc0 else np.zeros(0)
    return {"stages": stages, "term": term, "G0": G0, "g0": g0}


STAGE_ORDER = ("A", "B", "f", "Q", "S", "R", "q", "r", "C", "D", "d")


def stage_blocks(rec, nx, nu, nc):
    """A packed stage record -> {block: array in math layout} and 'pad': the doubles after d."""
    shapes = dict(A=(nx, nx), B=(nx, nu), f=(nx,), Q=(nx, nx), S=(nx, nu), R=(nu, nu), q=(nx,), r=(nu,), C=(nc, nx),
                  D=(nc, nu), d=(nc,))
    out, o = {}, 0
    for n in STAGE_ORDER:
        s = shapes[n]
        size = int(np.prod(s))
        a = np.asarray(rec[o:o + size])
        out[n] = a.reshape(s[::-1]).T if len(s) == 2 else a
        o += size
    out["pad"] = np.asarray(rec[o:])
    return out


def term_blocks(rec, nx, nct):
    out, o = {}, 0
    for n, s in (("Q", (nx, nx)), ("q", (nx,)), ("C", (nct, nx)), ("d", (nct,))):
        size = int(np.prod(s))
        a = np.asarray(rec[o:o + size])
        out[n] = a.reshape(s[::-1]).T if len(s) == 2 else a
        o += size
    return out


# ---------------------------------------------------------------------------------------------------------------------
# Line search (solver-proxddp.hxx:111-155, merit-function.hxx:13-104)
# ---------------------------------------------------------------------------------------------------------------------
def linear_step(cur, step, alpha):
    """results + alpha * step, element by element: one fused multiply-add, so the correctly rounded exact value."""
    cur, step = np.asarray(cur, dtype=np.float64), np.asarray(step, dtype=np.float64)
    a = Fraction(float(alpha))
    out = np.empty(cur.shape)
    for i in np.ndindex(cur.shape):
        out[i] = correctly_rounded(Fraction(float(cur[i])) + a * Fraction(float(step[i])))
    return out


def directional_derivative(Lxs, Lus, dxs, dus):
    """Lxs[0].dxs[0] + sum_i (Lxs[i+1].dxs[i+1] + Lus[i].dus[i])   (merit-function.hxx:82-101)."""
    terms = [(float(a), float(b)) for a, b in zip(np.ravel(Lxs), np.ravel(dxs))]
    terms += [(float(a), float(b)) for a, b in zip(np.ravel(Lus), np.ravel(dus))]
    return _bound(terms)


def al_value(cost, lam0, lams, vs, vsT, mudyn, mucstr):
    """cost + 1/2 (mucstr |lam_0|^2 + mudyn sum |lam_{i+1}|^2 + mucstr (sum |v_i|^2 + |v_N|^2))   (merit-function.hxx:
    41-65); ``cost`` None: no cost term.  The three sums of squares, the products by the penalties and the three
    additions: m = terms + 4."""
    mudyn, mucstr = float(mudyn), float(mucstr)
    terms = [] if cost is None else [(float(cost),)]
    terms += [(0.5, mucstr, float(l), float(l)) for l in np.ravel(lam0)]
    terms += [(0.5, mudyn, float(l), float(l)) for l in np.ravel(lams)]
    terms += [(0.5, mucstr, float(v), float(v)) for v in list(np.ravel(vs)) + list(np.ravel(vsT))]
    e, T, m = exact_sum(terms)
    return Bound(e, T, m + 4)
