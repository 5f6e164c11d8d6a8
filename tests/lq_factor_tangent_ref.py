"""Numpy restatement of ab2_gar_factor_tangent (include/aligator_b200/gar.h): the forward mode of the backward
recursion, from a tangent of the problem records to the tangents of the factorisation (FF, FB, VXX, VX, FFT, FBT).

Factor arrays as in lq_factor_adjoint_ref: ff [B][N][nu+nc+nx], fb [B][N][nu+nc+nx][nx], Vxx [B][N+1][nx][nx] (only
lower triangles are read), vx [B][N+1][nx], ffT [B][nct], fbT [B][nct][nx].  The tangent is a dict with any of stage
[B][N][srec], term [B][trec] (a missing or None key is zero; G0 and g0 do not enter).  The result has the factor
arrays' shapes, keyed ff, fb, vxx, vx, fft, fbt.

The tangent recursion runs backward in time, carrying Vd, vd (the tangents of Vxx_{t+1}, vx_{t+1}).  At the terminal
knot (Z_N = C_N / mu, z_N = d_N / mu):
    Zd_N = Cd_N / mu,  zd_N = dd_N / mu,  Vd_N = sym(Qd_N + Cd_N^T Z_N + C_N^T Zd_N),  vd_N = qd_N + Cd_N^T z_N + C_N^T zd_N
and per stage knot, with V' = Vxx_{t+1}, X = [[K, k], [Z, z]], Shat = S + A^T V' B, v+ = vx_{t+1} + V' f and
M = [[R + B^T V' B, D^T], [D, -mu I]]:
    vd+ = vd' + Vd' f + V' fd,  Shatd = Sd + Ad^T V' B + A^T Vd' B + A^T V' Bd,
    Rhatd = sym(Rd) + Bd^T V' B + B^T V' Bd + B^T Vd' B,  Qhatd = sym(Qd) + Ad^T V' A + A^T V' Ad + A^T Vd' A,
    rhatd = rd + Bd^T v+ + B^T vd+,  qhatd = qd + Ad^T v+ + A^T vd+
    [[Kd, kd], [Zd, zd]] = -M^-1 [[Rhatd K + Dd^T Z + Shatd^T, Rhatd k + Dd^T z + rhatd], [Dd K + Cd, Dd k + dd]]
    Ahatd = Ad + Bd K + B Kd,  ad = fd + Bd k + B kd
    Vd_t = sym(Qhatd + Shatd K + Shat Kd + Cd^T Z + C^T Zd),  vd_t = qhatd + Shatd k + Shat kd + Cd^T z + C^T zd
"""
from __future__ import annotations

import numpy as np

from lq_adjoint_ref import batched_solve, dtype_of, stage_offsets, term_offsets
from lq_factor_adjoint_ref import torch_factor


def _sym(M):
    return 0.5 * (M + np.swapaxes(M, -1, -2))


def _sym_lower(M):
    return np.tril(M) + np.swapaxes(np.tril(M, -1), -1, -2)


def factor_tangent(stage, term, ff, fb, Vxx, vx, ffT, fbT, dot, dims, mueq, solve=None):
    """Tangents of the factorisation along `dot`.  `mueq`: number or [B] array.  In the dtype of the inputs (see
    lq_adjoint_ref); `solve`: the 2-D solver for object arrays (None: np.linalg.solve)."""
    nx, nu, nc, nct, nc0, N = dims
    n = nu + nc
    B = np.asarray(term).shape[0]
    ty = dtype_of(stage, term, ff, fb, Vxx, vx, ffT, fbT, np.asarray(mueq), *dot.values())
    so, srec = stage_offsets(nx, nu, nc)
    to, trec = term_offsets(nx, nct)
    st = np.asarray(stage, dtype=ty).reshape(B, N, srec)
    tt = np.asarray(term, dtype=ty).reshape(B, -1)
    ds = np.zeros((B, N, srec), dtype=ty) if dot.get("stage") is None else \
        np.asarray(dot["stage"], ty).reshape(B, N, srec)
    dt = np.zeros(tt.shape, dtype=ty) if dot.get("term") is None else np.asarray(dot["term"], ty).reshape(tt.shape)
    blk = lambda rec, off, m, k: np.swapaxes(rec[..., off[0]:off[1]].reshape(*rec.shape[:-1], k, m), -1, -2)
    vec = lambda rec, off: rec[..., off[0]:off[1]]
    mu = np.broadcast_to(np.asarray(mueq, dtype=ty), (B,))
    V = _sym_lower(np.asarray(Vxx, dtype=ty))
    ff = np.asarray(ff, dtype=ty).reshape(B, N, n + nx)
    fb = np.asarray(fb, dtype=ty).reshape(B, N, n + nx, nx)
    vx = np.asarray(vx, dtype=ty).reshape(B, N + 1, nx)
    mv = lambda M, x: np.einsum("bij,bj->bi", M, x)
    T = lambda M: np.swapaxes(M, -1, -2)
    out = dict(ff=np.zeros((B, N, n + nx), dtype=ty), fb=np.zeros((B, N, n + nx, nx), dtype=ty),
               vxx=np.zeros((B, N + 1, nx, nx), dtype=ty), vx=np.zeros((B, N + 1, nx), dtype=ty))
    # terminal
    CN, dCN = blk(tt, to["C"], nct, nx), blk(dt, to["C"], nct, nx)
    ZN = np.asarray(fbT, dtype=ty).reshape(B, nct, nx)
    zN = np.asarray(ffT, dtype=ty).reshape(B, nct)
    dZN = dCN / mu[:, None, None]
    dzN = vec(dt, to["d"]) / mu[:, None]
    Vd = _sym(blk(dt, to["Q"], nx, nx) + T(dCN) @ ZN + T(CN) @ dZN)
    vd = vec(dt, to["q"]) + mv(T(dCN), zN) + mv(T(CN), dzN)
    out["vxx"][:, N], out["vx"][:, N] = Vd, vd
    out["fft"], out["fbt"] = dzN, dZN
    for t in range(N - 1, -1, -1):
        r, d = st[:, t], ds[:, t]
        A, Bm, f = blk(r, so["A"], nx, nx), blk(r, so["B"], nx, nu), vec(r, so["f"])
        S, R, C, D = blk(r, so["S"], nx, nu), blk(r, so["R"], nu, nu), blk(r, so["C"], nc, nx), blk(r, so["D"], nc, nu)
        dA, dB, df = blk(d, so["A"], nx, nx), blk(d, so["B"], nx, nu), vec(d, so["f"])
        dQ, dS, dR = _sym(blk(d, so["Q"], nx, nx)), blk(d, so["S"], nx, nu), _sym(blk(d, so["R"], nu, nu))
        dq, dr = vec(d, so["q"]), vec(d, so["r"])
        dC, dD, dd = blk(d, so["C"], nc, nx), blk(d, so["D"], nc, nu), vec(d, so["d"])
        Vp = V[:, t + 1]
        K, Z, k, z = fb[:, t, :nu], fb[:, t, nu:n], ff[:, t, :nu], ff[:, t, nu:n]
        Sh = S + T(A) @ Vp @ Bm
        vplus = vx[:, t + 1] + mv(Vp, f)
        # products
        dvplus = vd + mv(Vd, f) + mv(Vp, df)
        dSh = dS + T(dA) @ Vp @ Bm + T(A) @ Vd @ Bm + T(A) @ Vp @ dB
        dRh = dR + T(dB) @ Vp @ Bm + T(Bm) @ Vp @ dB + T(Bm) @ Vd @ Bm
        dQh = dQ + T(dA) @ Vp @ A + T(A) @ Vp @ dA + T(A) @ Vd @ A
        drh = dr + mv(T(dB), vplus) + mv(T(Bm), dvplus)
        dqh = dq + mv(T(dA), vplus) + mv(T(A), dvplus)
        # solve
        M = np.zeros((B, n, n), dtype=ty)
        M[:, :nu, :nu] = _sym_lower(R + T(Bm) @ Vp @ Bm)
        M[:, nu:, :nu] = D
        M[:, :nu, nu:] = T(D)
        M[:, nu:, nu:] = -mu[:, None, None] * np.eye(nc)
        Yu = np.concatenate([dRh @ K + T(dD) @ Z + T(dSh), (mv(dRh, k) + mv(T(dD), z) + drh)[..., None]], -1)
        Yc = np.concatenate([dD @ K + dC, (mv(dD, k) + dd)[..., None]], -1)
        X = -batched_solve(solve, M, np.concatenate([Yu, Yc], 1))
        dK, dk, dZ, dz = X[:, :nu, :nx], X[:, :nu, nx], X[:, nu:, :nx], X[:, nu:, nx]
        # closed loop
        dAh = dA + dB @ K + Bm @ dK
        da = df + mv(dB, k) + mv(Bm, dk)
        out["fb"][:, t] = np.concatenate([dK, dZ, dAh], 1)
        out["ff"][:, t] = np.concatenate([dk, dz, da], -1)
        # value
        Vd = _sym(dQh + dSh @ K + Sh @ dK + T(dC) @ Z + T(C) @ dZ)
        vd = dqh + mv(dSh, k) + mv(Sh, dk) + mv(T(dC), z) + mv(T(C), dz)
        out["vxx"][:, t], out["vx"][:, t] = Vd, vd
    return out


def jvp(stage, term, case, mu, dot):
    """(factorisation, its tangent) by torch.func.jvp through torch_factor."""
    import torch
    f = lambda s, t: torch_factor(s, t, case, mu)
    fac, tan = torch.func.jvp(f, (torch.tensor(stage), torch.tensor(term)),
                              (torch.tensor(dot["stage"]), torch.tensor(dot["term"])))
    return {k: v.numpy() for k, v in fac.items()}, {k: v.numpy() for k, v in tan.items()}
