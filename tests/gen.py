"""Problem generators and an independent dense-KKT cross-check for the tests.

Shapes/distributions follow the reference's test fixtures
(tests/gar/test_util.cpp:14-76, tests/test_util.hpp:18-23) and SURVEY.md §8(d);
the reference's by-value-RNG / libc-rand quirks are deliberately NOT replicated
(every knot draws fresh numbers from a seeded numpy Generator).
"""
from __future__ import annotations

import numpy as np

from aligator_b200.lqr import LqrKnot, LqrProblem


def wishart(rng, n, p):
    root = rng.standard_normal((n, p))
    return root @ root.T


def generate_knot(rng, nx, nu, nc, nth=0, singular=False, nx2=None, conditioned=False,
                  control_rows=False):
    """tests/gar/test_util.cpp:14-55.  ``conditioned`` uses A = I + 0.1 N/sqrt(nx)
    (SURVEY §8d) instead of A ~ U[-1,1]; ``control_rows`` uses C=0, D=I rows with a
    random half zeroed (inactive box rows) instead of C=I."""
    k = LqrKnot(nx, nu, nc, nx2, nth)
    nx2 = k.nx2
    qsr = wishart(rng, nx + nu, nx + nu + 1) / max(nx, nu)
    k.Q[:] = qsr[:nx, :nx]
    k.S[:] = qsr[:nx, nx:]
    if singular:
        k.Q[:] = wishart(rng, nx, int(0.8 * (nx + nu)))
    k.R[:] = qsr[nx:, nx:]
    k.R[np.diag_indices(nu)] *= 1 + 1e-6
    k.q[:] = rng.uniform(-1, 1, nx)
    k.r[:] = rng.uniform(-1, 1, nu)
    if conditioned:
        k.A[:] = np.eye(nx2, nx) + 0.1 * rng.standard_normal((nx2, nx)) / np.sqrt(nx)
    else:
        k.A[:] = rng.uniform(-1, 1, (nx2, nx))
    k.B[:] = rng.uniform(-1, 1, (nx2, nu))
    k.f[:] = rng.standard_normal(nx2)
    if nc > 0:
        if control_rows and nu > 0:
            k.D[:] = np.eye(nc, nu)
            mask = rng.uniform(size=nc) < 0.5
            k.D[mask, :] = 0.0
            k.d[:] = rng.uniform(-1, 1, nc)
            k.d[mask] = 0.0
        else:
            k.C[:] = np.eye(nc, nx)
            k.d[:] = rng.uniform(-1, 1, nc)
    if nth > 0:
        k.Gx[:] = rng.standard_normal((nx, nth))
        k.Gu[:] = rng.standard_normal((nu, nth))
        k.Gth[:] = wishart(rng, nth, nth + 2)
        k.gamma[:] = rng.standard_normal(nth)
    return k


def generate_lq_problem(rng, x0, horz, nx, nu, nth=0, nc=0, singular=True, conditioned=False,
                        control_rows=False, term_nc=None):
    """tests/gar/test_util.cpp:57-76: `horz` stage knots + a terminal knot with
    nu=0 (non-singular), G0 = -I, g0 = x0."""
    knots = [generate_knot(rng, nx, nu, nc, nth, singular, conditioned=conditioned,
                           control_rows=control_rows) for _ in range(horz)]
    tnc = nc if term_nc is None else term_nc
    knots.append(generate_knot(rng, nx, 0, tnc, nth, False, conditioned=conditioned))
    p = LqrProblem(knots, nx)
    p.g0[:] = x0
    p.G0[:] = -np.eye(nx)
    return p


def lqr_dense_kkt(problem, mueq):
    """Full dense KKT matrix and rhs with the x' = A x + B u + f convention
    (E = -I), unknown order [lbda0, (x_t, u_t, v_t, lbda_{t+1})_t]; mirrors
    tests/gar/test_util.hpp:91-165.  Solve K z = -rhs."""
    st = problem.stages
    N = problem.horizon
    nc0 = problem.nc0
    n = nc0 + sum(k.nx + k.nu + k.nc for k in st) + sum(st[t].nx2 for t in range(N))
    K = np.zeros((n, n))
    rhs = np.zeros(n)
    nx0 = st[0].nx
    K[:nc0, nc0:nc0 + nx0] = problem.G0
    K[nc0:nc0 + nx0, :nc0] = problem.G0.T
    rhs[:nc0] = problem.g0
    idx = nc0
    offs = []
    for t, m in enumerate(st):
        nx, nu, nc = m.nx, m.nu, m.nc
        nb = nx + nu + nc
        offs.append(idx)
        blk = np.zeros((nb, nb))
        blk[:nx, :nx] = m.Q
        blk[:nx, nx:nx + nu] = m.S
        blk[nx:nx + nu, :nx] = m.S.T
        blk[nx:nx + nu, nx:nx + nu] = m.R
        blk[nx + nu:, :nx] = m.C
        blk[:nx, nx + nu:] = m.C.T
        blk[nx + nu:, nx:nx + nu] = m.D
        blk[nx:nx + nu, nx + nu:] = m.D.T
        blk[nx + nu:, nx + nu:] = -mueq * np.eye(nc)
        K[idx:idx + nb, idx:idx + nb] = blk
        rhs[idx:idx + nx] = m.q
        rhs[idx + nx:idx + nx + nu] = m.r
        rhs[idx + nx + nu:idx + nb] = m.d
        if t != N:
            r0 = idx + nb
            K[r0:r0 + m.nx2, idx:idx + nx] = m.A
            K[r0:r0 + m.nx2, idx + nx:idx + nx + nu] = m.B
            K[idx:idx + nx, r0:r0 + m.nx2] = m.A.T
            K[idx + nx:idx + nx + nu, r0:r0 + m.nx2] = m.B.T
            # -I coupling with x_{t+1}
            c0 = r0 + m.nx2
            K[r0:r0 + m.nx2, c0:c0 + m.nx2] = -np.eye(m.nx2)
            K[c0:c0 + m.nx2, r0:r0 + m.nx2] = -np.eye(m.nx2)
            rhs[r0:r0 + m.nx2] = m.f
            idx += nb + m.nx2
    return K, rhs, offs


def lqr_dense_solve(problem, mueq):
    """Independent solution of the whole LQ problem by one dense solve."""
    K, rhs, offs = lqr_dense_kkt(problem, mueq)
    z = np.linalg.solve(K, -rhs)
    st = problem.stages
    N = problem.horizon
    nc0 = problem.nc0
    xs, us, vs, lbdas = [], [], [], [z[:nc0].copy()]
    for t, m in enumerate(st):
        o = offs[t]
        xs.append(z[o:o + m.nx].copy())
        if not (t == N and m.nu == 0):
            us.append(z[o + m.nx:o + m.nx + m.nu].copy())
        vs.append(z[o + m.nx + m.nu:o + m.nx + m.nu + m.nc].copy())
        if t != N:
            nb = m.nx + m.nu + m.nc
            lbdas.append(z[o + nb:o + nb + m.nx2].copy())
    return xs, us, vs, lbdas


# ---------------------------------------------------------------------------
# Packed uniform-dims batches in the product's layout (include/aligator_b200/gar.h)
#   stage record [A | B | f | Q | S | R | q | r | C | D | d]   term [Q | q | C | d]
# ---------------------------------------------------------------------------
def stage_record(k):
    F = lambda a: np.asarray(a).ravel(order="F")
    return np.concatenate([F(k.A), F(k.B), F(k.f), F(k.Q), F(k.S), F(k.R), F(k.q), F(k.r),
                           F(k.C), F(k.D), F(k.d)])


def term_record(k):
    F = lambda a: np.asarray(a).ravel(order="F")
    return np.concatenate([F(k.Q), F(k.q), F(k.C), F(k.d)])


def pack_problems(problems):
    """list of uniform-dims LqrProblem (terminal knot nu=0) -> packed arrays."""
    p0 = problems[0]
    N = p0.horizon
    stage = np.stack([np.stack([stage_record(p.stages[t]) for t in range(N)]) if N > 0
                      else np.zeros((0, 0)) for p in problems])
    term = np.stack([term_record(p.stages[N]) for p in problems])
    G0 = np.stack([np.asarray(p.G0).ravel(order="F") for p in problems])
    g0 = np.stack([np.asarray(p.g0) for p in problems])
    return (np.ascontiguousarray(stage), np.ascontiguousarray(term),
            np.ascontiguousarray(G0), np.ascontiguousarray(g0))


def generate_batch(seed, batch, N, nx, nu, nc=0, nct=0, style="conditioned", control_rows=None):
    """SURVEY §8(d) synthetic inputs, instance b seeded (seed, b)."""
    if control_rows is None:
        control_rows = nc > 0
    probs = []
    for b in range(batch):
        rng = np.random.default_rng([seed, b])
        x0 = rng.standard_normal(nx)
        probs.append(generate_lq_problem(
            rng, x0, N, nx, nu, 0, nc, singular=False,
            conditioned=(style == "conditioned"), control_rows=control_rows, term_nc=nct))
    return probs


def rel_fro(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    den = np.linalg.norm(b.ravel())
    num = np.linalg.norm((a - b).ravel())
    return num / den if den > 0 else num


def make_pivoting(probs):
    """Force Bunch-Kaufman interchanges on UNconstrained knots: R = diag([[1,1.8],[1.8,4]], I)
    (SPD, but |a_00| < alpha*colmax, and the row test then picks an interchange with row 1)
    and weak B, so Rhat = R + B^T V B keeps the pattern.  Exercises the general-algorithm
    fallback of the CUDA fast path."""
    for p in probs:
        for k in p.stages[:-1]:
            nu = k.nu
            R = np.eye(nu)
            R[:2, :2] = [[1.0, 1.8], [1.8, 4.0]]
            k.R[:] = R
            k.B *= 0.02
            k.S *= 0.0
    return probs


def make_2x2_pivots(probs):
    """Force 2x2 Bunch-Kaufman pivots on control-constrained knots: a light control cost
    (R = 1e-3 I, S = 0, weak B so Rhat = R + B^T V B stays small) against fully active rows
    D = I makes |a_kk| < alpha*colmax, fails the row test too (rowmax = 1) and leaves
    |a_imax,imax| = mu < alpha*rowmax: the pivot is the 2x2 block {k, nu + k}
    (core/bunchkaufman.hpp:61-83).  Needs nc >= 1."""
    for p in probs:
        for k in p.stages[:-1]:
            nu, nc = k.nu, k.nc
            assert nc >= 1
            k.R[:] = 1e-3 * np.eye(nu)
            k.S[:] = 0.0
            k.B *= 0.01
            k.C[:] = 0.0
            k.D[:] = np.eye(nc, nu)
            k.d[:] = np.linspace(-0.5, 0.5, nc)
    return probs


def general_initial_condition(probs, nc0, seed):
    """Replace G0 = -I, g0 = x0 by nc0 Gaussian rows G0 (any nc0 in [0, nx]) and a Gaussian g0, as a state
    manifold's G0 = -Jdiff would be.  Each problem gets `cond_G0`, the 2-norm condition number of its G0 (1 when
    nc0 = 0)."""
    for b, p in enumerate(probs):
        rng = np.random.default_rng([seed, b, nc0])
        nx = p.stages[0].nx
        p.G0 = np.asfortranarray(rng.standard_normal((nc0, nx)))
        p.g0 = rng.standard_normal(nc0)
        p.cond_G0 = float(np.linalg.cond(p.G0)) if nc0 else 1.0
    return probs


def make_homogeneous(probs):
    """q = r = f = d = g0 = 0 with every other input left as it is: the solution is exactly zero."""
    for p in probs:
        for k in p.stages:
            for name in ("q", "r", "f", "d"):
                getattr(k, name)[:] = 0.0
        p.g0[:] = 0.0
    return probs


def scale_instances(probs, exponents, mueq):
    """Instance b times c_b = 2**exponents[b]: Q, S, R, q, r, C, D, d, the parametric blocks Gx, Gu, Gv, Gth,
    gamma (empty when nth = 0), G0 and g0 scaled (A, B, f kept), and mu_b = c_b * mueq.  Every saddle-point system
    of instance b is then exactly c_b times the original one.  Returns (scaled copies, [batch] per-instance mu)."""
    out = []
    for p, s in zip(probs, exponents):
        q = p.copy()
        c = 2.0 ** int(s)
        for k in q.stages:
            for name in ("Q", "S", "R", "q", "r", "C", "D", "d", "Gx", "Gu", "Gv", "Gth", "gamma"):
                getattr(k, name)[...] *= c
        q.G0 *= c
        q.g0 *= c
        out.append(q)
    return out, np.array([2.0 ** int(s) * mueq for s in exponents])


def kkt_condition(probs, Vxx, mueq, tmax=8):
    """max over (sampled) knots of cond([[Rhat, D^T],[D, -mu I]]) with Rhat = R + B^T V' B: the factor
    by which two correct fp64 solvers may differ on K, k, Z, z (SURVEY Appendix C).
    Vxx: [B][N+1][nx][nx] (from the oracle)."""
    worst = 1.0
    for b, p in enumerate(probs):
        N = p.horizon
        for t in list(range(min(N, tmax))) + list(range(max(N - tmax, 0), N)):
            k = p.stages[t]
            if k.nc == 0:
                continue
            V = np.tril(Vxx[b, t + 1]) + np.tril(Vxx[b, t + 1], -1).T
            Rh = k.R + k.B.T @ V @ k.B
            M = np.block([[Rh, k.D.T], [k.D, -mueq * np.eye(k.nc)]])
            worst = max(worst, np.linalg.cond(M))
    return worst
