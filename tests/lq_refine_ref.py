"""Numpy restatement of ab2_gar_refine / ab2_gar_refine_many (include/aligator_b200/gar.h): iterative refinement of a
solution estimate z of K z = -h on a given factorisation, with resolve (lq_resolve_ref) as the correction solver.

    r = K z + h,   delta = resolve(r) = -K^-1 r,   z <- z + delta

`residual` writes r in resolve's rhs layouts (keys q, r, d, dN, g0, f), the rows the kernel sums; h is the
problem's own vectors (h = None) or a dict of right-hand sides [nrhs][B][...] (a missing or None key is zero).
Solutions are dicts of arrays [nrhs][B][...] with keys xs, us, vs, vsT, lam0, lams.
"""
from __future__ import annotations

import numpy as np

import lq_resolve_ref as rref
from lq_adjoint_ref import stage_offsets, term_offsets


def own_rhs(stage, term, g0, dims):
    """The problem's own vectors as one right-hand side [1][B][...] in resolve's rhs layouts."""
    nx, nu, nc, nct, nc0, N = dims
    B = np.asarray(term).shape[0]
    so, srec = stage_offsets(nx, nu, nc)
    to, _ = term_offsets(nx, nct)
    st = np.asarray(stage, dtype=np.float64).reshape(B, N, srec)
    tt = np.asarray(term, dtype=np.float64).reshape(B, -1)
    vec = lambda name: st[..., so[name][0]:so[name][1]]
    q = np.concatenate([vec("q"), tt[:, None, to["q"][0]:to["q"][1]]], axis=1)
    h = dict(q=q, r=vec("r"), d=vec("d"), dN=tt[:, to["d"][0]:to["d"][1]],
             g0=np.asarray(g0, dtype=np.float64).reshape(B, nc0), f=vec("f"))
    return {k: v[None].copy() for k, v in h.items()}


def residual(stage, term, G0, g0, z, h, dims, mueq):
    """r = K z + h for every right-hand side (Q and R used as stored).  `mueq`: number or [B] array."""
    nx, nu, nc, nct, nc0, N = dims
    B = np.asarray(term).shape[0]
    nrhs = np.asarray(z["xs"]).shape[0]
    h = own_rhs(stage, term, g0, dims) if h is None else rref.full_rhs(h, dims, B, nrhs)
    so, srec = stage_offsets(nx, nu, nc)
    to, _ = term_offsets(nx, nct)
    st = np.asarray(stage, dtype=np.float64).reshape(B, N, srec)
    tt = np.asarray(term, dtype=np.float64).reshape(B, -1)
    blk = lambda rec, off, m, n: np.swapaxes(rec[..., off[0]:off[1]].reshape(*rec.shape[:-1], n, m), -1, -2)
    mu = np.broadcast_to(np.asarray(mueq, dtype=np.float64), (B,))
    G = np.swapaxes(np.asarray(G0, dtype=np.float64).reshape(B, nx, nc0), -1, -2)  # [B][nc0][nx]
    x, u, v, l = (np.asarray(z[k], dtype=np.float64) for k in ("xs", "us", "vs", "lams"))
    vT, l0 = np.asarray(z["vsT"], dtype=np.float64), np.asarray(z["lam0"], dtype=np.float64)
    mv = lambda M, y: np.einsum("btik,jbtk->jbti", M, y)   # M y
    mtv = lambda M, y: np.einsum("btki,jbtk->jbti", M, y)  # M^T y
    r = {k: np.array(h[k], dtype=np.float64) for k in rref.RHS}
    if N > 0:
        A, Bm, Q = blk(st, so["A"], nx, nx), blk(st, so["B"], nx, nu), blk(st, so["Q"], nx, nx)
        S, R = blk(st, so["S"], nx, nu), blk(st, so["R"], nu, nu)
        C, D = blk(st, so["C"], nc, nx), blk(st, so["D"], nc, nu)
        xt, xn = x[:, :, :N], x[:, :, 1:]
        lp = np.concatenate([np.zeros_like(l[:, :, :1]), l[:, :, :-1]], axis=2)  # lambda_t (t = 0: none)
        r["q"][:, :, :N] += mv(Q, xt) + mv(S, u) + mtv(C, v) + mtv(A, l) - lp
        r["q"][:, :, 0] += np.einsum("bci,jbc->jbi", G, l0)
        r["r"] += mtv(S, xt) + mv(R, u) + mtv(D, v) + mtv(Bm, l)
        r["d"] += mv(C, xt) + mv(D, u) - mu[None, :, None, None] * v
        r["f"] += mv(A, xt) + mv(Bm, u) - xn
    QN, CN = blk(tt, to["Q"], nx, nx), blk(tt, to["C"], nct, nx)
    xN = x[:, :, N]
    r["q"][:, :, N] += np.einsum("bik,jbk->jbi", QN, xN) + np.einsum("bci,jbc->jbi", CN, vT)
    r["q"][:, :, N] += -l[:, :, N - 1] if N > 0 else np.einsum("bci,jbc->jbi", G, l0)
    r["dN"] += np.einsum("bck,jbk->jbc", CN, xN) - mu[None, :, None] * vT
    r["g0"] += np.einsum("bci,jbi->jbc", G, x[:, :, 0])
    return r


def inf_norms(r):
    """[nrhs][B] = max |r| over every row of each right-hand side and instance."""
    nrhs, B = r["q"].shape[:2]
    m = np.zeros((nrhs, B))
    for v in r.values():
        if v.size:
            m = np.maximum(m, np.abs(v.reshape(nrhs, B, -1)).max(axis=-1))
    return m


def refine(stage, term, G0, g0, fb, fbT, Vxx, z, h, dims, mueq, steps):
    """`steps` refinement steps of z (copied) on the factorisation (fb, fbT, Vxx); returns (z, norms [nrhs][B][steps+1])."""
    z = {k: np.array(v, dtype=np.float64) for k, v in z.items()}
    nrhs = z["xs"].shape[0]
    norms = []
    for _ in range(steps):
        r = residual(stage, term, G0, g0, z, h, dims, mueq)
        norms.append(inf_norms(r))
        dz = rref.resolve(stage, term, G0, fb, fbT, Vxx, r, dims, mueq, nrhs)
        for k in z:
            z[k] += dz[k]
    norms.append(inf_norms(residual(stage, term, G0, g0, z, h, dims, mueq)))
    return z, np.stack(norms, axis=-1)
