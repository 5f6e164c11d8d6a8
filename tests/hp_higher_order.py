"""References for the Hessian-vector product of lq_solve_higher (DESIGN section 2p) at the bar of DESIGN section 5.

The loss is L(z) = sum_k <w_k, z_k> + 1/2 <w_k, z_k * z_k> over the solution fields z_k, so its cotangent is
c = w + w * z.  Along a data direction pdot (symmetric Q, R, Q_N) the HVP is the derivative of the gradient records of L:

* `hvp_hp`: extended precision, independent of the composition the device runs.  The gradient records of L at
  p + h pdot are hp_reference's (the extended-precision recursion of the displaced problem, z; the same recursion on
  the problem with its vectors replaced by -c, w = K^-1 c; lq_adjoint_ref.grad_records(z, w)), and the HVP is their
  central difference at TANGENT_DPS digits, checked against the difference at 2h as hp_reference.tangent_problem does.
* `hvp_fp64`: the numpy fp64 composition on the oracle's solves, m = resolve(c), zdot = resolve(rho(pdot; z)),
  mdot = resolve(w * zdot + rho_K(pdot; m)), Gdot = Gr(mdot; z) + Gr_K(m; zdot): its error against `hvp_hp` is e_ref.
"""
import numpy as np

import hp_reference as hp
import lq_adjoint_ref as aref
import lq_resolve_ref as rref
import lq_tangent_ref as tref
from test_higher_order_oracle import grad_modes, rho_modes
from test_hp_derivatives import oracle_solution

KEYS = aref.KEYS
RECS = ("stage", "term", "G0", "g0")


def _solve_with_vectors(p, mueq, pdot, h, vec):
    """hp_reference.solve_problem of p + h pdot with every vector replaced by `vec` (extended precision, one
    instance, keys q [N+1][nx], r, d, f [N][.], dN, g0 as resolve's right-hand side)."""
    displace = hp._displace

    def replaced(p_, st, G0, g0, pdot_, h_):
        st, G0, _ = displace(p_, st, G0, g0, pdot_, h_)
        N = p_.horizon
        for t in range(N):
            st[t]["q"], st[t]["r"], st[t]["d"], st[t]["f"] = vec["q"][t], vec["r"][t], vec["d"][t], vec["f"][t]
        st[N]["q"], st[N]["d"] = vec["q"][N], vec["dN"]
        return st, G0, vec["g0"]
    hp._displace = replaced
    try:
        return hp.solve_problem(p, mueq, pdot, h)
    finally:
        hp._displace = displace


def _grad_records(p, mueq, w, pdot, h):
    """Extended-precision gradient records of L at p + h pdot (one instance; w: the loss weights, [1][...] object)."""
    d6 = hp.dims_of(p)
    z = hp.solution_dict([hp.solve_problem(p, mueq, pdot, h)])
    c = {k: w[k] + w[k] * z[k] for k in KEYS}
    vec = dict(q=-c["xs"][0], r=-c["us"][0], d=-c["vs"][0], dN=-c["vsT"][0], g0=-c["lam0"][0], f=-c["lams"][0])
    adj = hp.solution_dict([_solve_with_vectors(p, mueq, pdot, h, vec)])
    return aref.grad_records(z, adj, d6)


def hvp_hp(probs, mueq, W, dot):
    """Extended-precision HVP records of the batch (fp64-rounded, [B][...]): W the loss weights and dot the direction,
    [B][...] fp64 dicts."""
    out = []
    for b, p in enumerate(probs):
        with hp.MP.workdps(hp.TANGENT_DPS):
            w = {k: hp.mpa(np.asarray(W[k])[b:b + 1]) for k in KEYS}
            pd = {k: np.asarray(v)[b] for k, v in dot.items()}

            def central(step):
                plus, minus = _grad_records(p, mueq, w, pd, step), _grad_records(p, mueq, w, pd, -step)
                return {k: (plus[k] - minus[k]) / (2 * step) for k in RECS}, plus

            hh = hp.MP.mpf(hp.TANGENT_STEP)
            (d1, g), (d2, _) = central(hh), central(2 * hh)
            for k in RECS:
                scale = max(hp._norm(d1[k]), hp._norm(d2[k]), hp._norm(g[k]))
                assert hp._norm(d1[k] - d2[k]) <= hp.SELF_CHECK * scale, (k, float(hp._norm(d1[k] - d2[k]) / scale))
                if d1[k].size:
                    small = np.vectorize(lambda v: abs(v) <= hp.NOISE * scale, otypes=[bool])(d1[k])
                    d1[k] = np.where(small, hp._ZERO, d1[k])
            out.append({k: hp.to64(v) for k, v in d1.items()})
    return {k: np.concatenate([o[k] for o in out]) for k in RECS}


def _rhs(v):
    return dict(q=v["xs"], r=v["us"], d=v["vs"], dN=v["vsT"], g0=v["lam0"], f=v["lams"])


def hvp_fp64(recs, d6, mueq, W, dot):
    """The fp64 composition of the HVP on the oracle's solves ([B][...])."""
    res = lambda v: oracle_solution(rref.replaced_records(*recs, _rhs(v), d6), d6, mueq)
    one = lambda v: {k: x[None] for k, x in v.items()}
    z = oracle_solution(recs, d6, mueq)
    m = res({k: W[k] + W[k] * z[k] for k in KEYS})
    zd = res(tref.rho(dot, z, d6))
    rk = rho_modes(1, d6, one(dot), one(m), False)
    md = res({k: W[k] * zd[k] + rk[k][0] for k in KEYS})
    return {k: v[0] for k, v in grad_modes(1, d6, one(md), one(z), True, one(m), one(zd)).items()}
