"""Numpy restatement of ab2_gar_resolve (include/aligator_b200/gar.h): the vector half of the Riccati recursion on a
given factorisation, for many right-hand sides.

    z = resolve(h) = -K^-1 h

is the solution of the LQ problem with its vectors replaced by h.  The matrices are read from the stage / terminal
records (A, B, S, R, C, D, C_N), G0, and the factorisation of a backward pass: fb [B][N][nu+nc+nx][nx] (= [K; Z; Ahat]),
fbT [B][nct][nx] and Vxx [B][N+1][nx][nx] (row index first; only lower triangles are read).  Right-hand sides and
solutions are dicts of arrays [nrhs][B][...]: h keys q, r, d, dN, g0, f (a missing or None key is zero), z keys
xs, us, vs, vsT, lam0, lams as in lq_adjoint_ref.
"""
from __future__ import annotations

import numpy as np

from lq_adjoint_ref import stage_offsets, term_offsets

RHS = ("q", "r", "d", "dN", "g0", "f")
SOL = ("xs", "us", "vs", "vsT", "lam0", "lams")


def rhs_shapes(dims, B):
    nx, nu, nc, nct, nc0, N = dims
    return dict(q=(B, N + 1, nx), r=(B, N, nu), d=(B, N, nc), dN=(B, nct), g0=(B, nc0), f=(B, N, nx))


def full_rhs(h, dims, B, nrhs):
    return {k: np.zeros((nrhs,) + s) if h.get(k) is None else np.asarray(h[k], dtype=np.float64).reshape((nrhs,) + s)
            for k, s in rhs_shapes(dims, B).items()}


def _sym_lower(M):
    return np.tril(M) + np.swapaxes(np.tril(M, -1), -1, -2)


def resolve(stage, term, G0, fb, fbT, Vxx, h, dims, mueq, nrhs):
    """z = -K^-1 h by the kernel's algebra (vx_t = (qhat + Shat k) + C^T z in the reference's order).  `mueq`: number or
    [B] array."""
    nx, nu, nc, nct, nc0, N = dims
    B = np.asarray(term).shape[0]
    h = full_rhs(h, dims, B, nrhs)
    so, srec = stage_offsets(nx, nu, nc)
    to, _ = term_offsets(nx, nct)
    st = np.asarray(stage, dtype=np.float64).reshape(B, N, srec)
    tt = np.asarray(term, dtype=np.float64).reshape(B, -1)
    blk = lambda rec, off, m, n: np.swapaxes(rec[..., off[0]:off[1]].reshape(*rec.shape[:-1], n, m), -1, -2)
    mu = np.broadcast_to(np.asarray(mueq, dtype=np.float64), (B,))
    V = _sym_lower(np.asarray(Vxx, dtype=np.float64))
    fb = np.asarray(fb, dtype=np.float64)
    z = {k: np.zeros((nrhs,) + s) for k, s in zip(SOL, rhs_shapes(dims, B).values())}
    ks = np.zeros((nrhs, B, N, nu + nc))
    avec = np.zeros((nrhs, B, N, nx))
    vxs = np.zeros((nrhs, B, N + 1, nx))
    CN = blk(tt, to["C"], nct, nx)
    zN = h["dN"] / mu[None, :, None]
    vx = h["q"][:, :, N] + np.einsum("bci,jbc->jbi", CN, zN)
    vxs[:, :, N] = vx
    for t in range(N - 1, -1, -1):
        Bm, R, D = blk(st[:, t], so["B"], nx, nu), blk(st[:, t], so["R"], nu, nu), blk(st[:, t], so["D"], nc, nu)
        A, S, C = blk(st[:, t], so["A"], nx, nx), blk(st[:, t], so["S"], nx, nu), blk(st[:, t], so["C"], nc, nx)
        Vp = V[:, t + 1]
        f, r, d, q = h["f"][:, :, t], h["r"][:, :, t], h["d"][:, :, t], h["q"][:, :, t]
        vp = vx + np.einsum("bik,jbk->jbi", Vp, f)
        Rh = _sym_lower(R + np.swapaxes(Bm, -1, -2) @ Vp @ Bm)
        KKT = np.zeros((B, nu + nc, nu + nc))
        KKT[:, :nu, :nu] = Rh
        KKT[:, nu:, :nu] = D
        KKT[:, :nu, nu:] = np.swapaxes(D, -1, -2)
        KKT[:, nu:, nu:] = -mu[:, None, None] * np.eye(nc)
        w = np.concatenate([r + np.einsum("bki,jbk->jbi", Bm, vp), d], axis=-1)
        kz = -np.linalg.solve(KKT[None], w[..., None])[..., 0]
        ks[:, :, t] = kz
        avec[:, :, t] = f + np.einsum("bic,jbc->jbi", Bm, kz[..., :nu])
        k, zt = kz[..., :nu], kz[..., nu:]
        qh = q + np.einsum("bki,jbk->jbi", A, vp)
        sk = np.einsum("bic,jbc->jbi", S, k) + np.einsum("bki,jbk->jbi", A, np.einsum("bkl,blc,jbc->jbk", Vp, Bm, k))
        vx = (qh + sk) + np.einsum("bci,jbc->jbi", C, zt)
        vxs[:, :, t] = vx
    M = np.zeros((B, nx + nc0, nx + nc0))
    M[:, :nx, :nx] = V[:, 0]
    G = np.swapaxes(np.asarray(G0, dtype=np.float64).reshape(B, nx, nc0), -1, -2)
    M[:, nx:, :nx] = G
    M[:, :nx, nx:] = np.swapaxes(G, -1, -2)
    s0 = -np.linalg.solve(M[None], np.concatenate([vx, h["g0"]], axis=-1)[..., None])[..., 0]
    x = s0[..., :nx]
    z["xs"][:, :, 0] = x
    z["lam0"] = s0[..., nx:]
    for t in range(N):
        F = fb[:, t]
        z["us"][:, :, t] = ks[:, :, t, :nu] + np.einsum("bcx,jbx->jbc", F[:, :nu], x)
        z["vs"][:, :, t] = ks[:, :, t, nu:] + np.einsum("bcx,jbx->jbc", F[:, nu:nu + nc], x)
        x = avec[:, :, t] + np.einsum("bcx,jbx->jbc", F[:, nu + nc:], x)
        z["xs"][:, :, t + 1] = x
        z["lams"][:, :, t] = vxs[:, :, t + 1] + np.einsum("bik,jbk->jbi", V[:, t + 1], x)
    z["vsT"] = zN + np.einsum("bcx,jbx->jbc", np.asarray(fbT, dtype=np.float64).reshape(B, nct, nx), x)
    return z


def replaced_records(stage, term, G0, g0, hj, dims):
    """The problem's records with every vector replaced by ONE right-hand side hj (dict of [B][...] arrays, None is
    zero): what the oracle's full solve of the replaced problem takes."""
    from lq_adjoint_ref import adjoint_records
    B = np.asarray(term).shape[0]
    hj = {k: v[0] for k, v in full_rhs({k: None if v is None else np.asarray(v)[None] for k, v in hj.items()},
                                       dims, B, 1).items()}
    cot = dict(xs=-hj["q"], us=-hj["r"], vs=-hj["d"], vsT=-hj["dN"], lam0=-hj["g0"], lams=-hj["f"])
    return adjoint_records(stage, term, G0, g0, cot, dims)


def random_rhs(rng, dims, B, nrhs):
    return {k: rng.standard_normal((nrhs,) + s) for k, s in rhs_shapes(dims, B).items()}


def replaced_problems(probs, hj):
    """Copies of the LqrProblem list `probs` with every vector replaced by ONE right-hand side hj (dict of [B][...]
    arrays, None is zero), for solvers that take problem objects (tests/hp_reference.py)."""
    out = []
    for b, p in enumerate(probs):
        q = p.copy()
        N = q.horizon
        get = lambda k, *i: 0.0 if hj.get(k) is None else np.asarray(hj[k])[(b,) + i]
        for t in range(N):
            k = q.stages[t]
            k.q[:], k.r[:], k.d[:], k.f[:] = get("q", t), get("r", t), get("d", t), get("f", t)
        q.stages[N].q[:] = get("q", N)
        q.stages[N].d[:] = get("dN")
        q.g0[:] = get("g0")
        out.append(q)
    return out
