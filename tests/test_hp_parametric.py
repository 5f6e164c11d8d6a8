"""The extended-precision restatement of parametric problems and of leg mode (tests/hp_reference.py:
solve_parametric, solve_legs) pinned by identities that do not run the recursion they check, and the oracle measured
against it.

- Where Gv = 0 the problem at a fixed theta is the plain problem with q += Gx theta, r += Gu theta: the parametric
  gains, value functions and rollout are the plain ones of that shifted problem.
- The envelope theorem: thGrad and thHess are the first and second theta-derivatives of the optimal value.
- Leg mode reproduces the serial solution: the condensed system is the exact Schur complement of the legs.
- With Gv != 0 and nc > 0 the reference's Vxt is not the exact theta-derivative (DESIGN §4); the restatement follows
  the reference, and the identity visibly misses."""
import functools

import numpy as np
import pytest

import gen
import hp_reference as hp
import lq_adjoint_ref as aref
import lq_cases

IDENTITY = 1e-30


def _maxrel(a, b):
    """Largest |a - b| over the largest |b| (extended precision, object arrays)."""
    a, b = np.ravel(a), np.ravel(b)
    if not b.size:
        return 0.0
    return float(max(abs(x - y) for x, y in zip(a, b)) / max(max(abs(y) for y in b), hp.MP.mpf(1e-300)))


def dyadic_problem(seed, N, nx, nu, nc, nct, nth):
    """make_problem with Gx, Gu on the 2^-20 grid, so that Gx theta and Gu theta are exact in fp64 for a theta of
    quarters: the shifted problem is then formed exactly."""
    p = lq_cases.make_problem(seed, N, nx, nu, nc, nct, nth)
    for k in p.stages:
        k.Gx[...] = np.round(k.Gx * 2.0 ** 20) / 2.0 ** 20
        k.Gu[...] = np.round(k.Gu * 2.0 ** 20) / 2.0 ** 20
    return p


def shift(p, theta):
    """The data direction (hp_reference._displace, step 1) that moves q_t by Gx_t theta and r_t by Gu_t theta."""
    nx, nu, nc, nct, nc0, N = hp.dims_of(p)
    so, srec = aref.stage_offsets(nx, nu, nc)
    to, trec = aref.term_offsets(nx, nct)
    stage, term = np.zeros((N, srec)), np.zeros(trec)
    for t in range(N):
        k = p.stages[t]
        stage[t, so["q"][0]:so["q"][1]] = exact(k.Gx, theta)
        stage[t, so["r"][0]:so["r"][1]] = exact(k.Gu, theta)
    term[to["q"][0]:to["q"][1]] = exact(p.stages[N].Gx, theta)
    return dict(stage=stage, term=term)


def exact(G, theta):
    """G theta in fp64, asserted exact."""
    v = G @ theta
    assert all(a == b for a, b in zip(hp.mpa(v), hp.mpa(G) @ hp.mpa(theta))), "G theta is not exact in fp64"
    return v


# (nx, nu, nc, nct, nth, N, nc0, mueq)
SHAPES = [(4, 2, 2, 0, 3, 6, 4, 1e-3), (5, 3, 0, 2, 5, 4, 5, 1e-8), (6, 2, 1, 1, 2, 3, 2, 1e-3), (3, 1, 0, 0, 1, 1, 0, 1e-8),
          (4, 2, 2, 2, 2, 0, 4, 1e-3)]
SIDS = ["nx%d_nu%d_nc%d_nct%d_nth%d_N%d_nc0%d" % s[:7] for s in SHAPES]


@functools.lru_cache(maxsize=None)
def shaped(shape):
    nx, nu, nc, nct, nth, N, nc0, mueq = shape
    p = dyadic_problem(sum(shape[:7]), N, nx, nu, nc, nct, nth)
    if nc0 != nx:
        gen.general_initial_condition([p], nc0, 11)
    thetas = [np.eye(nth)[j] for j in range(nth)] + [np.random.default_rng(5).integers(-16, 17, nth) / 4.0]
    return p, thetas


@pytest.mark.parametrize("shape", SHAPES, ids=SIDS)
def test_parametric_outputs_are_those_of_the_shifted_problem(shape):
    """Gv = 0: k + Kth theta, z + Zth theta, a + Yth theta, vx + Vxt theta and the rollout at theta equal the plain
    solve of the problem with q += Gx theta, r += Gu theta, to 1e-30, for theta = e_j and one theta of quarters."""
    nx, nu, nc, nct, nth, N, nc0, mueq = shape
    p, thetas = shaped(shape)
    worst = 0.0
    for theta in thetas:
        h = hp.solve_parametric(p, mueq, theta)
        s = hp.solve_problem(p, mueq, shift(p, theta), 1)
        th = hp.mpa(theta)
        for t in range(N):
            worst = max(worst, _maxrel(h["ff"][t] + h["fth"][t] @ th, s["ff"][t]), _maxrel(h["fb"][t], s["fb"][t]))
        for t in range(N + 1):
            worst = max(worst, _maxrel(h["vx"][t] + h["Vxt"][t] @ th, s["vx"][t]), _maxrel(h["Vxx"][t], s["Vxx"][t]))
        for k in ("xs", "us", "vs", "vsT", "lbd0", "lbdas"):
            worst = max(worst, _maxrel(h[k], s[k]))
    print("\nshifted-problem identity, worst relative residual: %.1e" % worst)
    assert worst <= IDENTITY


@pytest.mark.parametrize("shape", SHAPES, ids=SIDS)
def test_theta_gradient_and_hessian_by_the_envelope_theorem(shape):
    """Gv = 0: thGrad = sum_t (gamma_t + Gx_t^T x_t + Gu_t^T u_t) on the theta-free rollout and thHess = sum_t (Gth_t +
    Gx_t^T X_t + Gu_t^T U_t), X, U the rollout's theta-columns (rollout at e_j minus the theta-free one), to 1e-30."""
    nx, nu, nc, nct, nth, N, nc0, mueq = shape
    p, _ = shaped(shape)
    h0 = hp.solve_parametric(p, mueq)
    cols = [hp.solve_parametric(p, mueq, np.eye(nth)[j]) for j in range(nth)]
    grad, hess = hp.zeros(nth), hp.zeros(nth, nth)
    for t, k in enumerate(p.stages):
        Gx, Gu = hp.mpa(k.Gx), hp.mpa(k.Gu)
        grad = grad + hp.mpa(k.gamma) + Gx.T @ h0["xs"][t]
        hess = hess + hp.mpa(k.Gth)
        for j, c in enumerate(cols):
            hess[:, j] = hess[:, j] + Gx.T @ (c["xs"][t] - h0["xs"][t])
        if t < N:
            grad = grad + Gu.T @ h0["us"][t]
            for j, c in enumerate(cols):
                hess[:, j] = hess[:, j] + Gu.T @ (c["us"][t] - h0["us"][t])
    e = (_maxrel(h0["thGrad"], grad), _maxrel(h0["thHess"], hess))
    print("\nenvelope theorem, thGrad %.1e thHess %.1e" % e)
    assert max(e) <= IDENTITY


# (nx, nu, nc, nct, nc0, N, legs, mueq): 2, 3, 4 and 8 legs, horizons that do not split evenly, nc > 0, nct > 0
LEG_SHAPES = [(4, 2, 0, 0, 4, 11, 2, 1e-8), (4, 2, 2, 0, 4, 13, 3, 1e-3), (5, 3, 2, 2, 2, 9, 4, 1e-2),
              (3, 2, 0, 0, 3, 10, 8, 1e-8), (6, 3, 1, 2, 0, 17, 3, 1e-3), (4, 2, 0, 1, 1, 7, 8, 1e-8)]
LIDS = ["nx%d_nu%d_nc%d_nct%d_nc0%d_N%d_legs%d" % s[:7] for s in LEG_SHAPES]


def leg_problem(shape):
    nx, nu, nc, nct, nc0, N, T, mueq = shape
    probs = gen.generate_batch(300 + N + T, 1, N, nx, nu, nc, nct)
    if nc0 != nx:
        gen.general_initial_condition(probs, nc0, 12)
    return probs[0]


@pytest.mark.parametrize("shape", LEG_SHAPES, ids=LIDS)
def test_legs_reproduce_the_serial_solution(shape):
    """The leg restatement's xs, us, vs, lambda (leg heads from the condensed solve, the rest from the legs' rollouts)
    equal the serial extended-precision solution to 1e-30."""
    nx, nu, nc, nct, nc0, N, T, mueq = shape
    p = leg_problem(shape)
    h, s = hp.solve_legs(p, mueq, T), hp.solve_problem(p, mueq)
    e = max(_maxrel(h[k], s[k]) for k in ("xs", "us", "vs", "vsT", "lbd0", "lbdas"))
    print("\nlegs vs serial, worst relative residual: %.1e" % e)
    assert e <= IDENTITY
    assert list(h["param"]) == [t < hp.get_work(N, T - 1, T)[0] for t in range(N + 1)]


# well-conditioned cases: Gv = 0, nc = nct = 0 or a large mu
ORACLE_PARAM = [(5, 2, 0, 0, 3, 7, 5, 1e-8), (6, 3, 0, 0, 6, 8, 6, 1e-8), (4, 2, 2, 0, 4, 10, 4, 1e-1),
                (5, 2, 0, 0, 1, 1, 2, 1e-8)]
ORACLE_LEGS = [(4, 2, 0, 0, 4, 11, 3, 1e-8), (6, 3, 0, 0, 6, 20, 4, 1e-8), (3, 2, 0, 0, 3, 10, 8, 1e-8)]


@pytest.mark.parametrize("shape", ORACLE_PARAM, ids=["nx%d_nu%d_nc%d_nct%d_nth%d_N%d_nc0%d" % s[:7] for s in ORACLE_PARAM])
def test_oracle_parametric_within_the_floor(shape):
    """On well-conditioned parametric problems every family of the oracle -- gains, value functions with their theta
    terms, kkt0.fth, thGrad, thHess and the rollout at theta -- is within 64 u of the restatement."""
    nx, nu, nc, nct, nth, N, nc0, mueq = shape
    probs = [lq_cases.make_problem([sum(shape[:7]), b], N, nx, nu, nc, nct, nth) for b in range(2)]
    if nc0 != nx:
        gen.general_initial_condition(probs, nc0, 13)
    thetas = np.random.default_rng(6).standard_normal((2, nth))
    ref, _ = hp.solve_parametric_batch(probs, mueq, thetas)
    e = hp.error_families(lq_cases.oracle_parametric(probs, mueq, thetas), ref, nu, nc, N)
    print("\noracle, parametric %s: %s" % (shape, " ".join("%s %.1e" % kv for kv in e.items())))
    assert set(lq_cases.PARAM_KEYS[1:]) <= set(e) and max(e.values()) <= hp.FLOOR, e


@pytest.mark.parametrize("shape", ORACLE_LEGS, ids=["nx%d_nu%d_nc%d_nct%d_nc0%d_N%d_legs%d" % s[:7] for s in ORACLE_LEGS])
def test_oracle_legs_within_the_floor(shape):
    """On well-conditioned problems the oracle's ParallelRiccatiSolver -- every leg factor family, collapseFeedback and
    the rollout -- is within 64 u of the restatement."""
    nx, nu, nc, nct, nc0, N, T, mueq = shape
    p = leg_problem(shape)
    ref, _ = hp.solve_legs_batch([p], mueq, T)
    e = hp.error_families(lq_cases.oracle_legs([p], mueq, T), ref, nu, nc, N)
    print("\noracle, legs %s: %s" % (shape, " ".join("%s %.1e" % kv for kv in e.items())))
    assert {"Kth", "Vxt", "Vtt", "vt", "collapse", "xs"} <= set(e) and max(e.values()) <= hp.FLOOR, e


def test_gv_makes_vxt_miss_the_exact_derivative():
    """With Gv != 0 on knots with nc > 0 the reference's Vxt leaves out Z^T Gv (riccati-kernel.hxx:304-306, DESIGN §4):
    vx + Vxt theta misses the vx of the shifted problem (now also d += Gv theta) by far more than 64 u, while the same
    problem with Gv = 0 meets the identity."""
    nx, nu, nc, nct, nth, N, mueq = 4, 2, 2, 0, 3, 6, 1e-3
    p = lq_cases.make_problem(21, N, nx, nu, nc, nct, nth, gv=True)
    for k in p.stages:
        k.Gx[...], k.Gu[...] = 0.0, 0.0
        k.Gv[...] = np.round(k.Gv * 2.0 ** 20) / 2.0 ** 20
    theta = np.eye(nth)[0]
    h = hp.solve_parametric(p, mueq, theta)
    so, srec = aref.stage_offsets(nx, nu, nc)
    stage = np.zeros((N, srec))
    for t in range(N):
        stage[t, so["d"][0]:so["d"][1]] = exact(p.stages[t].Gv, theta)
    s = hp.solve_problem(p, mueq, dict(stage=stage), 1)
    th = hp.mpa(theta)
    miss = max(_maxrel(h["vx"][t] + h["Vxt"][t] @ th, s["vx"][t]) for t in range(N))
    print("\nGv != 0: worst relative miss of vx + Vxt theta: %.1e" % miss)
    assert miss >= 1e6 * hp.FLOOR
