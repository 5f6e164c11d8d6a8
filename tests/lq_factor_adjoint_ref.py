"""Numpy restatement of ab2_gar_factor_adjoint (include/aligator_b200/gar.h): the reverse mode of the backward
recursion, from cotangents of the factorisation (FF, FB, VXX, VX, FFT, FBT) to gradients of the problem records.

Factor arrays, as BatchedOracle.get() returns them: ff [B][N][nu+nc+nx] (= [k; z; a]), fb [B][N][nu+nc+nx][nx]
(= [K; Z; Ahat]), Vxx [B][N+1][nx][nx] (row index first; only lower triangles are read), vx [B][N+1][nx],
ffT [B][nct], fbT [B][nct][nx].  Cotangents are a dict with any of ff, fb, vxx, vx, fft, fbt in those shapes (a
missing or None key is zero).  Gradients are the records of lq_adjoint_ref.grad_records: stage [B][N][srec],
term [B][trec], G0 and g0 (zero: the initial condition does not enter the factorisation).

The reverse pass runs forward in time, carrying Vbar, vbar (the cotangents of Vxx_t, vx_t).  Per stage knot, with
V' = Vxx_{t+1}, v' = vx_{t+1}, X = [[K, k], [Z, z]], Shat = S + A^T V' B, v+ = v' + V' f and
M = [[R + B^T V' B, D^T], [D, -mu I]]:
    Kb = Kb0 + B^T Ahatb,  kb = kb0 + B^T ab,  Bb = Ahatb K^T + ab k^T,  Ab = Ahatb,  fb = ab
    Qb = Vbar,  qb = vbar,  Shatb = Vbar K^T + vbar k^T,  Kb += Shat^T Vbar,  kb += Shat^T vbar
    Cb = Z Vbar + z vbar^T,  Zb = Zb0 + C Vbar,  zb = zb0 + C vbar
    P = -M^-1 [[Kb, kb], [Zb, zb]];  Shatb += P_u[:, :nx]^T,  rb = P_u[:, nx],  Cb += P_c[:, :nx],  db = P_c[:, nx]
    Rb = sym(P_u X_u^T),  Db = P_c X_u^T + X_c P_u^T,  Sb = Shatb
    Ab += 2 V' A Qb + V' B Shatb^T + v+ qb^T,  Bb += 2 V' B Rb + V' A Shatb + v+ rb^T
    vb+ = A qb + B rb,  fb += V' vb+
    Vbar' = sym(Vxxb_{t+1}) + sym(A Qb A^T + B Rb B^T + A Shatb B^T + vb+ f^T),  vbar' = vxb_{t+1} + vb+
and at the terminal knot (Z_N = C_N / mu, z_N = d_N / mu):
    Zb = Zb0_N + C_N Vbar,  zb = zb0_N + C_N vbar,  C_Nb = Z_N Vbar + z_N vbar^T + Zb / mu,  d_Nb = zb / mu,
    Q_Nb = Vbar,  q_Nb = vbar.
"""
from __future__ import annotations

import numpy as np

from lq_adjoint_ref import batched_solve, dtype_of, stage_offsets, term_offsets

COT = ("ff", "fb", "vxx", "vx", "fft", "fbt")


def cot_shapes(dims, B):
    nx, nu, nc, nct, nc0, N = dims
    nr = nu + nc + nx
    return dict(ff=(B, N, nr), fb=(B, N, nr, nx), vxx=(B, N + 1, nx, nx), vx=(B, N + 1, nx), fft=(B, nct),
                fbt=(B, nct, nx))


def full_cot(cot, dims, B, dt=np.float64):
    return {k: np.zeros(s, dtype=dt) if cot.get(k) is None else np.asarray(cot[k], dtype=dt).reshape(s)
            for k, s in cot_shapes(dims, B).items()}


def random_cot(rng, dims, B):
    return {k: rng.standard_normal(s) for k, s in cot_shapes(dims, B).items()}


def _sym(M):
    return 0.5 * (M + np.swapaxes(M, -1, -2))


def _sym_lower(M):
    return np.tril(M) + np.swapaxes(np.tril(M, -1), -1, -2)


def _cm(M):
    """[..., m, n] -> column-major [..., m*n]."""
    return np.swapaxes(M, -1, -2).reshape(*M.shape[:-2], M.shape[-2] * M.shape[-1])


def factor_adjoint(stage, term, ff, fb, Vxx, vx, ffT, fbT, cot, dims, mueq, solve=None):
    """Gradient records of <cot, factorisation>.  `mueq`: number or [B] array.  In the dtype of the inputs (see
    lq_adjoint_ref); `solve`: the 2-D solver for object arrays (None: np.linalg.solve)."""
    nx, nu, nc, nct, nc0, N = dims
    n = nu + nc
    B = np.asarray(term).shape[0]
    dt = dtype_of(stage, term, ff, fb, Vxx, vx, ffT, fbT, np.asarray(mueq), *cot.values())
    c = full_cot(cot, dims, B, dt)
    so, srec = stage_offsets(nx, nu, nc)
    to, trec = term_offsets(nx, nct)
    st = np.asarray(stage, dtype=dt).reshape(B, N, srec)
    tt = np.asarray(term, dtype=dt).reshape(B, -1)
    blk = lambda rec, off, m, k: np.swapaxes(rec[..., off[0]:off[1]].reshape(*rec.shape[:-1], k, m), -1, -2)
    mu = np.broadcast_to(np.asarray(mueq, dtype=dt), (B,))
    V = _sym_lower(np.asarray(Vxx, dtype=dt))
    ff = np.asarray(ff, dtype=dt).reshape(B, N, n + nx)
    fb = np.asarray(fb, dtype=dt).reshape(B, N, n + nx, nx)
    vx = np.asarray(vx, dtype=dt).reshape(B, N + 1, nx)
    gs = np.zeros((B, N, srec), dtype=dt)
    gt = np.zeros((B, trec), dtype=dt)
    Vb = _sym(c["vxx"][:, 0])
    vb = c["vx"][:, 0].copy()
    mv = lambda M, x: np.einsum("bij,bj->bi", M, x)
    T = lambda M: np.swapaxes(M, -1, -2)
    outer = lambda a, b_: a[:, :, None] * b_[:, None, :]
    for t in range(N):
        r = st[:, t]
        A, Bm, f = blk(r, so["A"], nx, nx), blk(r, so["B"], nx, nu), r[:, so["f"][0]:so["f"][1]]
        S, R, C, D = blk(r, so["S"], nx, nu), blk(r, so["R"], nu, nu), blk(r, so["C"], nc, nx), blk(r, so["D"], nc, nu)
        Vp, vp = V[:, t + 1], vx[:, t + 1]
        K, Z, k, z = fb[:, t, :nu], fb[:, t, nu:n], ff[:, t, :nu], ff[:, t, nu:n]
        Xu = np.concatenate([K, k[..., None]], axis=-1)
        Xc = np.concatenate([Z, z[..., None]], axis=-1)
        Sh = S + T(A) @ Vp @ Bm
        vplus = vp + mv(Vp, f)
        Ahb, ab = c["fb"][:, t, n:], c["ff"][:, t, n:]
        # closed loop
        Kb = c["fb"][:, t, :nu] + T(Bm) @ Ahb
        kb = c["ff"][:, t, :nu] + mv(T(Bm), ab)
        Bb = Ahb @ T(K) + outer(ab, k)
        Ab = Ahb.copy()
        fbar = ab.copy()
        # value
        Qb, qb = Vb, vb
        Shb = Vb @ T(K) + outer(vb, k)
        Kb = Kb + T(Sh) @ Vb
        kb = kb + mv(T(Sh), vb)
        Cb = Z @ Vb + outer(z, vb)
        Zb = c["fb"][:, t, nu:n] + C @ Vb
        zb = c["ff"][:, t, nu:n] + mv(C, vb)
        # solve
        M = np.zeros((B, n, n), dtype=dt)
        M[:, :nu, :nu] = _sym_lower(R + T(Bm) @ Vp @ Bm)
        M[:, nu:, :nu] = D
        M[:, :nu, nu:] = T(D)
        M[:, nu:, nu:] = -mu[:, None, None] * np.eye(nc)
        Xb = np.concatenate([np.concatenate([Kb, kb[..., None]], -1), np.concatenate([Zb, zb[..., None]], -1)], 1)
        P = -batched_solve(solve, M, Xb)
        Pu, Pc = P[:, :nu], P[:, nu:]
        Shb = Shb + T(Pu[..., :nx])
        rb = Pu[..., nx]
        Cb = Cb + Pc[..., :nx]
        db = Pc[..., nx]
        Rb = _sym(Pu @ T(Xu))
        Db = Pc @ T(Xu) + Xc @ T(Pu)
        # products
        Ab = Ab + 2.0 * Vp @ A @ Qb + Vp @ Bm @ T(Shb) + outer(vplus, qb)
        Bb = Bb + 2.0 * Vp @ Bm @ Rb + Vp @ A @ Shb + outer(vplus, rb)
        vbp = mv(A, qb) + mv(Bm, rb)
        fbar = fbar + mv(Vp, vbp)
        blocks = dict(A=_cm(Ab), B=_cm(Bb), f=fbar, Q=_cm(Qb), S=_cm(Shb), R=_cm(Rb), q=qb, r=rb, C=_cm(Cb),
                      D=_cm(Db), d=db)
        for key, (a0, a1) in so.items():
            gs[:, t, a0:a1] = blocks[key]
        # carry
        G = A @ Qb @ T(A) + Bm @ Rb @ T(Bm) + A @ Shb @ T(Bm) + outer(vbp, f)
        Vb = _sym(c["vxx"][:, t + 1]) + _sym(G)
        vb = c["vx"][:, t + 1] + vbp
    # terminal
    CN = blk(tt, to["C"], nct, nx)
    ZN = np.asarray(fbT, dtype=dt).reshape(B, nct, nx)
    zN = np.asarray(ffT, dtype=dt).reshape(B, nct)
    ZNb = c["fbt"] + CN @ Vb
    zNb = c["fft"] + mv(CN, vb)
    CNb = ZN @ Vb + outer(zN, vb) + ZNb / mu[:, None, None]
    dNb = zNb / mu[:, None]
    tb = dict(Q=_cm(Vb), q=vb, C=_cm(CNb), d=dNb)
    for key, (a0, a1) in to.items():
        gt[:, a0:a1] = tb[key]
    return dict(stage=gs, term=gt, G0=np.zeros((B, nc0 * nx), dtype=dt), g0=np.zeros((B, nc0), dtype=dt))
