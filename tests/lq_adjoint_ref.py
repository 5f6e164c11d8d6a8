"""Numpy restatement of the adjoint of the LQ solve (ab2_gar_adjoint, include/aligator_b200/gar.h).

The LQ solution z solves K z = -h.  For a loss with cotangent zbar, w = K^-1 zbar is the solution of the same LQ
problem with the vectors replaced by minus the cotangent (`adjoint_records`), and the gradients are dh = -w and
dK = -w z^T read out of K's blocks (`grad_records`; the symmetric Q and R get the symmetric part).

Solutions and cotangents are dicts of batched arrays in the solver's output layouts: xs [B][N+1][nx], us [B][N][nu],
vs [B][N][nc], vsT [B][nct], lam0 [B][nc0], lams [B][N][nx] (lambda_1 .. lambda_N).  Records are the packed
[B][N][stage_record] / [B][term_record] / [B][nc0*nx] / [B][nc0] arrays of gar.h.

Every function here and in the other restatements (lq_tangent_ref, lq_factor_adjoint_ref, lq_factor_tangent_ref)
computes in the dtype of its inputs: float64, or object arrays of extended-precision numbers (tests/hp_reference.py),
for which every buffer is allocated as object and every linear solve goes through the `solve` hook.
"""
from __future__ import annotations

import numpy as np

KEYS = ("xs", "us", "vs", "vsT", "lam0", "lams")


def stage_offsets(nx, nu, nc, nth=0):
    """(start, end) of each block of a stage record, with the parametric tail when nth > 0, and the padded record
    length.  Mirrors csrc/lq_record.cuh (checked by test_record_layout.py)."""
    sizes = [("A", nx * nx), ("B", nx * nu), ("f", nx), ("Q", nx * nx), ("S", nx * nu), ("R", nu * nu), ("q", nx),
             ("r", nu), ("C", nc * nx), ("D", nc * nu), ("d", nc)]
    if nth:
        sizes += [("Gx", nx * nth), ("Gu", nu * nth), ("Gv", nc * nth), ("Gth", nth * nth), ("gamma", nth)]
    off, o = {}, 0
    for k, n in sizes:
        off[k] = (o, o + n)
        o += n
    return off, o + (o % 2)


def term_offsets(nx, nct, nth=0):
    """(start, end) of each block of a terminal record, with the parametric tail when nth > 0, and the record length."""
    sizes = [("Q", nx * nx), ("q", nx), ("C", nct * nx), ("d", nct)]
    if nth:
        sizes += [("Gx", nx * nth), ("Gv", nct * nth), ("Gth", nth * nth), ("gamma", nth)]
    off, o = {}, 0
    for k, n in sizes:
        off[k] = (o, o + n)
        o += n
    return off, o


def dtype_of(*arrays):
    """object when any input holds extended-precision numbers (an object array), else float64."""
    return object if any(getattr(a, "dtype", None) == object for a in arrays) else np.float64


def batched_solve(solve, M, X):
    """M^-1 X for stacks of systems M [..., n, n], X [..., n, m]: np.linalg.solve, or `solve` (a 2-D solver of object
    arrays, hp_reference.lu_solve) system by system."""
    if solve is None:
        return np.linalg.solve(M, X)
    lead = np.broadcast_shapes(M.shape[:-2], X.shape[:-2])
    M, X = np.broadcast_to(M, lead + M.shape[-2:]), np.broadcast_to(X, lead + X.shape[-2:])
    out = np.empty(lead + X.shape[-2:], dtype=object)
    for i in np.ndindex(*lead):
        out[i] = solve(M[i], X[i].copy()) if M.shape[-1] else X[i]
    return out


def _shapes(dims, B):
    nx, nu, nc, nct, nc0, N = dims
    return dict(xs=(B, N + 1, nx), us=(B, N, nu), vs=(B, N, nc), vsT=(B, nct), lam0=(B, nc0), lams=(B, N, nx))


def _full(cot, dims, B, dt=np.float64):
    """Cotangent dict with missing / None entries as zeros."""
    return {k: np.zeros(s, dtype=dt) if cot.get(k) is None else np.asarray(cot[k], dtype=dt).reshape(s)
            for k, s in _shapes(dims, B).items()}


def adjoint_records(stage, term, G0, g0, cot, dims):
    """The adjoint problem: the matrices of (stage, term, G0) and the vectors q, r, d, f, q_N, d_N, g0 = -cotangent."""
    nx, nu, nc, nct, nc0, N = dims
    B = term.shape[0]
    dt = dtype_of(stage, term, G0, *cot.values())
    c = _full(cot, dims, B, dt)
    so, srec = stage_offsets(nx, nu, nc)
    to, _ = term_offsets(nx, nct)
    st = np.array(stage, dtype=dt).reshape(B, N, srec)
    tt = np.array(term, dtype=dt).reshape(B, -1)
    for k, v in (("q", c["xs"][:, :N]), ("r", c["us"]), ("d", c["vs"]), ("f", c["lams"])):
        st[..., so[k][0]:so[k][1]] = -v
    tt[:, to["q"][0]:to["q"][1]] = -c["xs"][:, N]
    tt[:, to["d"][0]:to["d"][1]] = -c["vsT"]
    return st, tt, np.array(G0, dtype=dt).reshape(B, -1), -c["lam0"]


def _outer(a, b):
    return a[..., :, None] * b[..., None, :]


def _cm(M):
    """[..., m, n] -> column-major [..., m*n]."""
    return np.swapaxes(M, -1, -2).reshape(*M.shape[:-2], M.shape[-2] * M.shape[-1])


def grad_records(z, w, dims):
    """Gradient records from the primal solution z and the adjoint solution w (dicts of batched arrays)."""
    nx, nu, nc, nct, nc0, N = dims
    B = np.asarray(z["xs"]).shape[0]
    dt = dtype_of(*z.values(), *w.values())
    z, w = _full(z, dims, B, dt), _full(w, dims, B, dt)
    so, srec = stage_offsets(nx, nu, nc)
    to, trec = term_offsets(nx, nct)
    x, u, v, l = z["xs"][:, :N], z["us"], z["vs"], z["lams"]
    X, U, V, L = w["xs"][:, :N], w["us"], w["vs"], w["lams"]
    pair = lambda a, b, A, B_: -(_outer(A, b) + _outer(a, B_))  # -(A b^T + a B^T)
    blocks = dict(A=_cm(pair(l, x, L, X)), B=_cm(pair(l, u, L, U)), f=-L, Q=_cm(0.5 * pair(x, x, X, X)),
                  S=_cm(pair(x, u, X, U)), R=_cm(0.5 * pair(u, u, U, U)), q=-X, r=-U, C=_cm(pair(v, x, V, X)),
                  D=_cm(pair(v, u, V, U)), d=-V)
    st = np.zeros((B, N, srec), dtype=dt)
    for k, (a, b) in so.items():
        st[..., a:b] = blocks[k]
    xN, XN = z["xs"][:, N], w["xs"][:, N]
    tb = dict(Q=_cm(0.5 * pair(xN, xN, XN, XN)), q=-XN, C=_cm(pair(z["vsT"], xN, w["vsT"], XN)), d=-w["vsT"])
    tt = np.zeros((B, trec), dtype=dt)
    for k, (a, b) in to.items():
        tt[:, a:b] = tb[k]
    G0 = _cm(pair(z["lam0"], z["xs"][:, 0], w["lam0"], w["xs"][:, 0]))
    return dict(stage=st, term=tt, G0=G0, g0=-w["lam0"])


def solution_dict(sols, dims):
    """Per-instance (xs, us, vs, lbdas) lists of gen.lqr_dense_solve -> batched solution dict."""
    N = dims[5]
    cat = lambda a: np.concatenate([np.ravel(v) for v in a]) if len(a) else np.zeros(0)
    per = [dict(xs=cat(xs), us=cat(us[:N]), vs=cat(vs[:N]), vsT=np.ravel(vs[N]), lam0=np.ravel(lbdas[0]),
                lams=cat(lbdas[1:])) for xs, us, vs, lbdas in sols]
    return {k: np.stack([d[k] for d in per]).reshape(s) for k, s in _shapes(dims, len(sols)).items()}


def oracle_dict(o):
    """BatchedOracle.get() -> batched solution dict."""
    return dict(xs=o["xs"], us=o["us"], vs=o["vs"], vsT=o["vsT"], lam0=o["lbd0"], lams=o["lbdas"])
