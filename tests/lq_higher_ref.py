"""Numpy restatements of the streaming maps of the LQ solve's derivatives (DESIGN section 2p): the gradient records
Gr(y; z) of ab2_gar_adjoint_many (`grad_many`), and the two modes of ab2_gar_rho_many / ab2_gar_grad_many
(`rho_modes`, `grad_modes`: per-direction vectors, two terms, with and without the vector blocks, e)."""
import numpy as np

import lq_adjoint_ref as aref
import lq_tangent_ref as tref

KEYS = aref.KEYS
RECS = ("stage", "term", "G0", "g0")


def grad_many(z, y, d6):
    """Gradient records from z and y = resolve(zbar) (the kernel's formulas: dh = y, dK = y z^T, symmetric part of
    Q and R)."""
    nx, nu, nc, nct, nc0, N = d6
    so, srec = aref.stage_offsets(nx, nu, nc)
    to, trec = aref.term_offsets(nx, nct)
    B = z["xs"].shape[0]
    o, cm = aref._outer, aref._cm
    pair = lambda a, b, ya, yb: o(ya, b) + o(a, yb)  # y_a b^T + a y_b^T
    x, u, v, l = z["xs"][:, :N], z["us"], z["vs"], z["lams"]
    X, U, V, L = y["xs"][:, :N], y["us"], y["vs"], y["lams"]
    blocks = dict(A=cm(pair(l, x, L, X)), B=cm(pair(l, u, L, U)), f=L, Q=cm(0.5 * pair(x, x, X, X)),
                  S=cm(pair(x, u, X, U)), R=cm(0.5 * pair(u, u, U, U)), q=X, r=U, C=cm(pair(v, x, V, X)),
                  D=cm(pair(v, u, V, U)), d=V)
    st = np.zeros((B, N, srec))
    for k, (a, b) in so.items():
        st[..., a:b] = blocks[k]
    xN, XN = z["xs"][:, N], y["xs"][:, N]
    tb = dict(Q=cm(0.5 * pair(xN, xN, XN, XN)), q=XN, C=cm(pair(z["vsT"], xN, y["vsT"], XN)), d=y["vsT"])
    tt = np.zeros((B, trec))
    for k, (a, b) in to.items():
        tt[:, a:b] = tb[k]
    G0 = cm(pair(z["lam0"], z["xs"][:, 0], y["lam0"], y["xs"][:, 0]))
    return dict(stage=st, term=tt, G0=G0, g0=y["lam0"])


def _no_vectors(dot, d6):
    """The tangent records with their vector blocks (q, r, d, f, q_N, d_N, g0) zero: rho(., a) of it is rho_K."""
    nx, nu, nc, nct, nc0, N = d6
    so, _ = aref.stage_offsets(nx, nu, nc)
    to, _ = aref.term_offsets(nx, nct)
    out = {k: None if dot.get(k) is None else np.array(dot[k], dtype=np.float64) for k in RECS}
    if out["stage"] is not None:
        for k in ("f", "q", "r", "d"):
            out["stage"][..., so[k][0]:so[k][1]] = 0.0
    if out["term"] is not None:
        for k in ("q", "d"):
            out["term"][..., to[k][0]:to[k][1]] = 0.0
    out["g0"] = None
    return out


def _zero_vector_blocks(g, d6):
    """Gradient records with their vector blocks written 0: Gr_K from Gr."""
    return _no_vectors(g, d6) | {"g0": np.zeros_like(g["g0"])}


def _at(v, j):
    """Direction j of a dict of [nrhs][batch][...] arrays, or the dict itself when it is shared ([batch][...])."""
    return v if v.get("each") is False else {k: None if v.get(k) is None else v[k][j] for k in v if k != "each"}


def rho_modes(nrhs, d6, dot1, a1, vec=True, dot2=None, a2=None, e=None):
    """out_j = rho^(vec)(dot1_j; a1_j) + rho_K(dot2_j; a2_j) + e_j, per direction (the kernel's sum order: term 1,
    term 2, e).  A vector dict with each=False is shared."""
    outs = []
    for j in range(nrhs):
        d1 = {k: None if dot1.get(k) is None else dot1[k][j] for k in RECS}
        r = tref.rho(d1 if vec else _no_vectors(d1, d6), {k: _at(a1, j)[k] for k in KEYS}, d6)
        if dot2 is not None:
            d2 = _no_vectors({k: None if dot2.get(k) is None else dot2[k][j] for k in RECS}, d6)
            r2 = tref.rho(d2, {k: _at(a2, j)[k] for k in KEYS}, d6)
            r = {k: r[k] + r2[k] for k in KEYS}
        if e is not None:
            r = {k: r[k] + e[k][j] for k in KEYS}
        outs.append(r)
    return {k: np.stack([o[k] for o in outs]) for k in KEYS}


def grad_modes(nrhs, d6, y1, z1, vec=True, y2=None, z2=None):
    """out_j = Gr^(vec)(y1_j; z1_j) + Gr_K(y2_j; z2_j), per direction."""
    outs = []
    for j in range(nrhs):
        g = grad_many({k: _at(z1, j)[k] for k in KEYS}, {k: y1[k][j] for k in KEYS}, d6)
        if not vec:
            g = _zero_vector_blocks(g, d6)
        if y2 is not None:
            g2 = _zero_vector_blocks(grad_many({k: _at(z2, j)[k] for k in KEYS}, {k: y2[k][j] for k in KEYS}, d6), d6)
            g = {k: g[k] + g2[k] for k in RECS}
        outs.append(g)
    return {k: np.stack([o[k] for o in outs]) for k in RECS}
