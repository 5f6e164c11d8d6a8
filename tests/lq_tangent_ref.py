"""Numpy restatement of the tangent (forward mode) of the LQ solve (ab2_gar_tangent, include/aligator_b200/gar.h).

The LQ solution z solves K z = -h with K affine in the data, so along a data tangent pdot = (Kdot, hdot) the solution
moves by zdot = -K^-1 rho, rho = Kdot z + hdot: the solution of the same LQ problem with the vectors q, r, d, f, q_N,
d_N, g0 replaced by rho (`tangent_records`).  The tangent of Q and R enters through sym(.) = (. + .^T) / 2, which makes
this the exact transpose of lq_adjoint_ref.grad_records.

Tangents are dicts with any of stage [B][N][stage_record], term [B][term_record], G0 [B][nc0*nx] (column-major),
g0 [B][nc0] (a missing or None entry is zero); solutions are dicts in the layouts of lq_adjoint_ref.
"""
from __future__ import annotations

import numpy as np

from lq_adjoint_ref import _full, adjoint_records, dtype_of, stage_offsets, term_offsets


def _blk(rec, off, m, n):
    """Column-major m x n block of the batched records rec [..., record] at offset `off` = (start, end)."""
    a, b = off
    return np.swapaxes(rec[..., a:b].reshape(*rec.shape[:-1], n, m), -1, -2)


def _sym(M):
    return 0.5 * (M + np.swapaxes(M, -1, -2))


def _mv(M, y):
    return np.einsum("...ij,...j->...i", M, y)


def _mtv(M, y):
    return np.einsum("...ji,...j->...i", M, y)


def rho(dot, z, dims):
    """rho = Kdot z + hdot in the cotangent layout (xs, us, vs, vsT, lam0, lams) of lq_adjoint_ref."""
    nx, nu, nc, nct, nc0, N = dims
    B = np.asarray(z["xs"]).shape[0]
    dt = dtype_of(*z.values(), *dot.values())
    z = _full(z, dims, B, dt)
    so, srec = stage_offsets(nx, nu, nc)
    to, trec = term_offsets(nx, nct)
    get = lambda k, s: np.zeros(s, dtype=dt) if dot.get(k) is None else np.asarray(dot[k], dtype=dt).reshape(s)
    st, tt = get("stage", (B, N, srec)), get("term", (B, trec))
    G0, g0 = np.swapaxes(get("G0", (B, nx, nc0)), -1, -2), get("g0", (B, nc0))
    x, u, v, l = z["xs"][:, :N], z["us"], z["vs"], z["lams"]
    A, Bm, Q = _blk(st, so["A"], nx, nx), _blk(st, so["B"], nx, nu), _blk(st, so["Q"], nx, nx)
    S, R = _blk(st, so["S"], nx, nu), _blk(st, so["R"], nu, nu)
    C, D = _blk(st, so["C"], nc, nx), _blk(st, so["D"], nc, nu)
    vec = lambda k: st[..., so[k][0]:so[k][1]]
    out = dict(
        us=vec("r") + _mtv(S, x) + _mv(_sym(R), u) + _mtv(D, v) + _mtv(Bm, l),
        vs=vec("d") + _mv(C, x) + _mv(D, u),
        lams=vec("f") + _mv(A, x) + _mv(Bm, u))
    xs = np.zeros((B, N + 1, nx), dtype=dt)
    xs[:, :N] = vec("q") + _mv(_sym(Q), x) + _mv(S, u) + _mtv(C, v) + _mtv(A, l)
    xN, vN = z["xs"][:, N], z["vsT"]
    QN, CN = _blk(tt, to["Q"], nx, nx), _blk(tt, to["C"], nct, nx)
    xs[:, N] = tt[:, to["q"][0]:to["q"][1]] + _mv(_sym(QN), xN) + _mtv(CN, vN)
    xs[:, 0] += _mtv(G0, z["lam0"])
    out["xs"] = xs
    out["vsT"] = tt[:, to["d"][0]:to["d"][1]] + _mv(CN, xN)
    out["lam0"] = g0 + _mv(G0, z["xs"][:, 0])
    return out


def tangent_records(stage, term, G0, g0, dot, z, dims):
    """The tangent problem: the matrices of (stage, term, G0) and the vectors q, r, d, f, q_N, d_N, g0 = rho.  Its
    solution is zdot."""
    r = rho(dot, z, dims)
    return adjoint_records(stage, term, G0, g0, {k: -v for k, v in r.items()}, dims)
