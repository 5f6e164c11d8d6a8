"""The exact element-wise references of the inner-iteration kernels (tests/exact_inner_ref.py) and the extended-precision
FDDP backward pass (hp_reference.fddp_backward_pass), on the CPU.

* The exact-arithmetic helpers (tests/exact_bounds.py) against plain Fraction arithmetic.
* The references reproduce the hand cases of the numpy restatements exactly, and the restatements (fp64) land within the
  references' bounds on random cases.
* The bar rejects planted errors that the restatement-based checks accept.
* The FDDP reference satisfies the recursion's defining equations to 1e-30 and agrees with oracle/fddp.py to 64 u."""
import math
from fractions import Fraction

import numpy as np
import pytest

import exact_inner_ref as xr
import gen
import hp_reference as hp
from exact_bounds import U, correctly_rounded, exact_sum, same_bits, within
from oracle import fddp as of
from oracle import linesearch as ols
from oracle import lq_assemble as olq
from oracle import proxddp_inner as pin
from inner_cases import fddp_args, fddp_case, hand_case, hand_gradient_inputs, random_inputs

INF = np.inf


# ---------------------------------------------------------------------------------------------------------------------
# exact_bounds
# ---------------------------------------------------------------------------------------------------------------------
def test_exact_sum_matches_fraction_arithmetic():
    rng = np.random.default_rng(1)
    for n in (1, 2, 7, 300):
        a = rng.standard_normal(n) * 2.0 ** rng.integers(-200, 200, n)
        b = rng.standard_normal(n) * 2.0 ** rng.integers(-200, 200, n)
        terms = [(float(x), float(y)) for x, y in zip(a, b)] + [(1.5,), (float(a[0]), Fraction(1, 3))]
        e, T, m = exact_sum(terms)
        want = sum((Fraction(x) * Fraction(y) for x, y in zip(a, b)), Fraction(0)) + Fraction(3, 2) + Fraction(a[0]) / 3
        wantT = sum((abs(Fraction(x) * Fraction(y)) for x, y in zip(a, b)), Fraction(0)) + Fraction(3, 2) + abs(Fraction(a[0])) / 3
        assert (e, T, m) == (want, wantT, n + 2)


def test_correctly_rounded_and_within():
    one = Fraction(1)
    assert correctly_rounded(one + U) == 1.0                      # a tie: to even
    assert correctly_rounded(one + 3 * U) == 1.0 + 4 * float(U)   # a tie: to even, upwards
    assert correctly_rounded(one + U + Fraction(1, 2 ** 80)) == 1.0 + 2 * float(U)
    assert correctly_rounded(Fraction(2) ** 1024) == math.inf and correctly_rounded(-Fraction(2) ** 1024) == -math.inf
    assert correctly_rounded(Fraction(3, 2 ** 1076)) == 2.0 ** -1074   # rounds into the subnormals
    # a fp64 dot product lies within the bound; one that is off by more does not
    rng = np.random.default_rng(2)
    x, y = rng.standard_normal(200), rng.standard_normal(200)
    e, T, m = exact_sum([(float(a), float(b)) for a, b in zip(x, y)])
    assert within(float(np.dot(x, y)), e, T, m)
    assert not within(float(e) + 1e-10 * float(T), e, T, m)
    assert not within(math.nan, e, T, m)
    assert same_bits(0.0, 0.0) and not same_bits(0.0, -0.0) and same_bits(math.nan, -math.nan)


# ---------------------------------------------------------------------------------------------------------------------
# the references against the hand cases
# ---------------------------------------------------------------------------------------------------------------------
def _hand_mult_inputs(h):
    N = len(h["xs"]) - 1
    return dict(xs=np.array(h["xs"]), lam0=h["lams"][0], lams=np.array(h["lams"][1:]), vs=np.array(h["vs"][:N]),
                vsT=h["vs"][N], prev_vs=np.array(h["prev_vs"][:N]), prev_vsT=h["prev_vs"][N],
                init_value=h["init_value"], cval=np.array(h["cvals"][:N]), cval_N=h["cvals"][N],
                xnext=np.array(h["xnext"]))


def _restated_outputs(m, N, nx, nc):
    """The numpy restatement's results in the device's output layout."""
    return dict(slack=np.array(m["fs"][1:]).reshape(N, nx), lam0_plus=m["lams_plus"][0],
                lams_plus=np.array(m["lams_plus"][1:]).reshape(N, nx),
                shifted=np.array(m["shifted"][:N]).reshape(N, nc), shifted_N=m["shifted"][N],
                vs_plus=np.array(m["vs_plus"][:N]).reshape(N, nc), vsT_plus=m["vs_plus"][N],
                Lv=np.array(m["Lvs"][:N]).reshape(N, nc), Lv_N=m["Lvs"][N])


def _exact(w):
    return np.array([float(v.exact) if isinstance(v, xr.Bound) else v for v in np.ravel(w)]).reshape(np.shape(w))


def test_multipliers_reference_reproduces_the_hand_case():
    h = hand_case()
    m = pin.compute_multipliers(**h)
    got = _restated_outputs(m, 1, 2, 3)
    w = xr.multipliers(_hand_mult_inputs(h), got, h["lo"], h["hi"], h["loN"], h["hiN"], h["mu"], h["mu_dyn"])
    assert np.array_equal(w["slack"], [[10.0, 10.0]])
    assert np.array_equal(_exact(w["lam0_plus"]), [2.0, -2.0]) and np.array_equal(_exact(w["lams_plus"]), [[42.0, 40.0]])
    assert np.array_equal(_exact(w["shifted"]), [[0.5, 0.5, 1.0]]) and np.array_equal(w["vs_plus"], [[1.0, 1.0, 0.0]])
    assert np.array_equal(_exact(w["Lv"]), [[0.0, -0.5, 0.5]])
    assert np.array_equal(_exact(w["shifted_N"]), [-0.75]) and np.array_equal(w["vsT_plus"], [0.0])
    assert np.array_equal(_exact(w["Lv_N"]), [-1.5])
    assert w["prim"][0] <= 10 <= w["prim"][1] and float(w["prim"][1]) == 10.0
    assert xr.flag(got) == 1.0
    for k in ("slack", "lam0_plus", "lams_plus", "shifted", "shifted_N", "vs_plus", "vsT_plus", "Lv", "Lv_N"):
        assert not xr.failures(got[k], w[k]), k


def test_gradient_and_criterion_references_reproduce_the_hand_case():
    h, g = hand_case(), hand_gradient_inputs()
    inp = dict(lx=np.array(g["lx"]), lu=np.array(g["lu"]), lx_N=g["lx_N"], Jx=np.array(g["Jx"]), Ju=np.array(g["Ju"]),
               cJx=np.array(g["cJx"]), cJu=np.array(g["cJu"]), cJx_N=g["cJx_N"], G0=g["G0"], lam0=h["lams"][0],
               lams=np.array(h["lams"][1:]), vs=np.array(h["vs"][:1]), vsT=h["vs"][1])
    Lxs, Lus = xr.lagrangian_gradient(inp)
    assert np.array_equal(_exact(Lxs), [[3.5, 3.5], [5.0, -2.0]]) and np.array_equal(_exact(Lus), [[3.0]])
    Lxf, _ = xr.lagrangian_gradient(inp, force_initial_condition=True)
    assert np.array_equal(_exact(Lxf)[0], [0.0, 0.0]) and same_bits(Lxf[0, 0], 0.0)
    m = pin.compute_multipliers(**h)
    assert xr.criterion(_exact(Lxs), _exact(Lus), h["init_value"], np.array(m["fs"][1:]), np.array(m["Lvs"][:1]),
                        m["Lvs"][1]) == (5.0, 5.0)


def test_assembly_reference_reproduces_the_hand_case():
    inp = dict(Jx=np.array([[[1., 2.], [3., 4.]]]), Ju=np.array([[[5.], [6.]]]), slack=np.array([[.5, -.5]]),
               Lxx=np.array([[[2., 1.], [1., 3.]]]), Lxu=np.array([[[1.], [0.]]]), Luu=np.array([[[4.]]]),
               Lx=np.array([[1., 1.]]), Lu=np.array([[2.]]),
               cJx=np.array([[[1., 0.], [0., 2.]]]), cJu=np.array([[[1.], [3.]]]), Lv=np.array([[2., 4.]]),
               shifted=np.array([[0.3, -1.0]]), lo=np.array([np.inf, -np.inf]), hi=np.array([np.inf, 0.0]),
               Lxx_N=np.eye(2), Lx_N=np.array([1., 2.]), G0=-np.eye(2), g0=np.array([.1, .2]),
               Hxx0=np.array([[10., 0.], [0., 10.]]))
    p = xr.assemble(inp, 1, 2, 1, 2, 0, 2, 0.5, 10.0)
    k = p["stages"][0]
    assert np.array_equal(_exact(k["Q"]), [[12.5, 1.], [1., 13.5]]) and np.array_equal(_exact(k["R"]), [[4.5]])
    assert np.array_equal(k["C"], [[1., 0.], [0., 0.]]) and np.array_equal(k["D"], [[1.], [0.]])
    assert not np.signbit(k["C"][1]).any()
    assert np.array_equal(_exact(k["q"]), [1., 81.]) and np.array_equal(_exact(k["r"]), [122.])
    assert np.array_equal(_exact(p["term"]["Q"]), 1.5 * np.eye(2)) and np.array_equal(_exact(p["term"]["q"]), [1., 2.])
    assert np.array_equal(p["G0"], -np.eye(2)) and np.array_equal(p["g0"], [.1, .2])


def test_line_search_references_reproduce_the_hand_case():
    assert np.array_equal(xr.linear_step([1.0, 2.0, 0.0], [1.0, 0.0, 2.0], 0.5), [1.5, 2.0, 1.0])
    b = xr.directional_derivative([[2.0, 1.0], [1.0, 1.0]], [[4.0]], [[1.0, 0.0], [0.0, 2.0]], [[-1.0]])
    assert b.exact == 0 and b.T == 8
    v = xr.al_value(1.0, [1.0, 1.0], [[2.0, 0.0]], [[2.0]], [], 0.1, 10.0)
    assert v.exact == 1 + Fraction(1, 2) * (10 * 2 + Fraction(0.1) * 4 + 10 * 4)


def test_projection_follows_the_reference_comparisons():
    """z on the bound is not outside it; the sign of a zero and a NaN come out of std::min / std::max's comparisons."""
    nc = xr.normal_cone
    assert nc(1.0, -1.0, 1.0) == 0.0 and nc(-1.0, -1.0, 1.0) == 0.0 and nc(1.5, -1.0, 1.0) == 0.5
    assert same_bits(nc(-0.0, -INF, 0.0), 0.0)          # -0 - (-0) = +0
    assert same_bits(nc(0.0, -INF, -0.0), 0.0) and same_bits(nc(-0.0, -0.0, 0.0), 0.0)
    assert same_bits(nc(-0.0, INF, INF), -0.0)           # an equality row keeps z, sign included
    assert nc(3.0, 2.0, 2.0) == 1.0 and nc(2.0, 2.0, 2.0) == 0.0   # pinned box
    assert math.isnan(nc(math.nan, -1.0, 1.0)) and math.isnan(nc(-INF, -INF, 0.0)) and nc(INF, -1.0, 1.0) == INF
    assert not xr.active(1.0, -1.0, 1.0) and xr.active(1.0 + 2e-16 * 2, -1.0, 1.0) and xr.active(0.0, INF, INF)


# ---------------------------------------------------------------------------------------------------------------------
# the restatements land within the references' bounds
# ---------------------------------------------------------------------------------------------------------------------
def _assembled_blocks(prob, N):
    return {t: prob["stages"][t] for t in range(N)}, prob["term"]


@pytest.mark.parametrize("dims", [(3, 4, 2, 3, 2, 4), (4, 5, 3, 0, 0, 5), (0, 4, 2, 0, 2, 4), (2, 6, 3, 40, 33, 3)])
def test_assembly_restatement_within_the_reference(dims):
    N, nx, nu, nc, nct, nc0 = dims
    rng = np.random.default_rng(sum(dims))
    inp = random_inputs(rng, N, nx, nu, nc, nct, nc0, exact=True, init_hess=True)
    prob = olq.assemble_problem(inp, N, nx, nu, nc, nct, nc0)
    w = xr.assemble(inp, N, nx, nu, nc, nct, nc0, inp["preg"], inp["mu_inv"])
    for t in range(N):
        for n in xr.STAGE_ORDER:
            assert not xr.failures(prob["stages"][t][n], w["stages"][t][n]), (t, n)
    for n in ("Q", "q", "C", "d"):
        assert not xr.failures(prob["term"][n], w["term"][n]), n
    assert not xr.failures(prob["G0"], w["G0"]) and not xr.failures(prob["g0"], w["g0"])


def _random_mult(rng, N, nx, nc, nct, nc0):
    r = lambda *s: rng.standard_normal(s)
    inp = dict(xs=r(N + 1, nx), lam0=r(nc0), lams=r(N, nx), vs=r(N, nc), vsT=r(nct), prev_vs=r(N, nc),
               prev_vsT=r(nct), init_value=r(nc0), cval=r(N, nc), cval_N=r(nct), xnext=r(N, nx))
    kinds, kindsN = np.arange(nc) % 4, (np.arange(nct) + 1) % 4
    bnd = lambda k: (np.select([k == 0, k == 1, k == 2], [INF, -INF, -0.5], 0.25),
                     np.select([k == 0, k == 1, k == 2], [INF, 0.0, 0.5], 0.25))
    return inp, bnd(kinds), bnd(kindsN)


@pytest.mark.parametrize("dims", [(3, 4, 5, 2, 4), (5, 3, 0, 0, 3), (0, 3, 0, 3, 2), (2, 2, 37, 35, 2)])
def test_multiplier_and_gradient_restatements_within_the_reference(dims):
    N, nx, nc, nct, nc0 = dims
    nu = 2
    rng = np.random.default_rng(sum(dims))
    inp, (lo, hi), (loN, hiN) = _random_mult(rng, N, nx, nc, nct, nc0)
    mu, mu_dyn = 0.03, 0.007
    m = pin.compute_multipliers(list(inp["xs"]), [inp["lam0"]] + list(inp["lams"]), list(inp["vs"]) + [inp["vsT"]],
                                list(inp["prev_vs"]) + [inp["prev_vsT"]], inp["init_value"],
                                list(inp["cval"]) + [inp["cval_N"]], lo, hi, loN, hiN, mu, mu_dyn,
                                xnext=list(inp["xnext"]))
    got = _restated_outputs(m, N, nx, nc)
    w = xr.multipliers(inp, got, lo, hi, loN, hiN, mu, mu_dyn)
    for k in ("slack", "lam0_plus", "lams_plus", "shifted", "shifted_N", "vs_plus", "vsT_plus", "Lv", "Lv_N"):
        assert not xr.failures(got[k], w[k]), k
    assert w["prim"][0] <= Fraction(m["prim_infeas"]) <= w["prim"][1]
    assert xr.flag(got) == 1.0 and m["ok"]
    # the gradient, force off and on
    r = lambda *s: rng.standard_normal(s)
    g = dict(lx=r(N, nx), lu=r(N, nu), lx_N=r(nx), Jx=r(N, nx, nx), Ju=r(N, nx, nu), cJx=r(N, nc, nx), cJu=r(N, nc, nu),
             cJx_N=r(nct, nx), G0=r(nc0, nx), lam0=inp["lam0"], lams=inp["lams"], vs=inp["vs"], vsT=inp["vsT"])
    for force in (False, True):
        Lxs, Lus = pin.lagrangian_gradient(list(g["lx"]), list(g["lu"]), g["lx_N"], list(g["Jx"]), list(g["Ju"]),
                                           list(g["cJx"]), list(g["cJu"]), g["cJx_N"], g["G0"],
                                           [g["lam0"]] + list(g["lams"]), list(g["vs"]) + [g["vsT"]],
                                           force_initial_condition=force)
        wx, wu = xr.lagrangian_gradient(g, force)
        assert not xr.failures(np.array(Lxs), wx) and not xr.failures(np.array(Lus).reshape(N, nu), wu), force
        crit = pin.criterion(Lxs, Lus, m["fs"], m["Lvs"])
        assert xr.criterion(np.array(Lxs), np.array(Lus).reshape(N, nu), m["fs"][0], got["slack"], got["Lv"],
                            got["Lv_N"]) == crit


def test_line_search_restatements_within_the_reference():
    rng = np.random.default_rng(5)
    N, nx, nu = 40, 5, 3
    xs, dxs, us, dus = rng.standard_normal((N + 1, nx)), rng.standard_normal((N + 1, nx)), rng.standard_normal((N, nu)), rng.standard_normal((N, nu))
    alpha = 0.37
    tx = ols.try_linear_step(list(xs), list(us), [], [], list(dxs), list(dus), [], [], alpha)[0]
    # numpy rounds the product and the sum apart: within two roundings of the exact value; the fused one is exact
    for got, x, dx in zip(np.ravel(tx), np.ravel(xs), np.ravel(dxs)):
        e, T, m = exact_sum([(float(x),), (alpha, float(dx))])
        assert within(got, e, T, m)
    b = xr.directional_derivative(xs, us, dxs, dus)
    assert within(ols.directional_derivative(list(xs), list(us), list(dxs), list(dus)), *b)
    lam0, lams, vs, vsT = rng.standard_normal(3), rng.standard_normal((N, nx)), rng.standard_normal((N, 2)), rng.standard_normal(2)
    v = xr.al_value(1.25, lam0, lams, vs, vsT, 0.01, 7.0)
    assert within(ols.al_value(1.25, [lam0] + list(lams), list(vs) + [vsT], 0.01, 7.0, True), *v)


# ---------------------------------------------------------------------------------------------------------------------
# planted errors: the new bar rejects what the restatement-based checks accept
# ---------------------------------------------------------------------------------------------------------------------
def test_bar_rejects_a_1e12_error_in_one_S_entry():
    rng = np.random.default_rng(11)
    N, nx, nu, nc, nct, nc0 = 4, 4, 2, 3, 0, 4
    inp = random_inputs(rng, N, nx, nu, nc, nct, nc0)
    inp["mu_inv"] = 1e3                              # the constraint corrections in q, r set the scale at ~1e3
    import aligator_b200.gar as gar
    srec = gar.stage_record_doubles(nx, nu, nc)
    want = olq.pack(olq.assemble_problem(inp, N, nx, nu, nc, nct, nc0), N, nx, nu, nc, nct, srec)[0]
    got = want.copy()
    s0 = nx * nx + nx * nu + nx + nx * nx                 # offset of S in a record
    got[1, s0] *= 1 + 1e-12
    assert np.max(np.abs(got - want)) <= 1e-13 * np.abs(want).max()      # test_lq_assemble's check accepts it
    w = xr.assemble(inp, N, nx, nu, nc, nct, nc0, inp["preg"], inp["mu_inv"])
    assert not xr.failures(xr.stage_blocks(want[1], nx, nu, nc)["S"], w["stages"][1]["S"])
    assert xr.failures(xr.stage_blocks(got[1], nx, nu, nc)["S"], w["stages"][1]["S"])


def test_bar_rejects_a_linear_step_one_ulp_off():
    rng = np.random.default_rng(12)
    x, dx, alpha = rng.standard_normal(500), rng.standard_normal(500), 0.37
    want = xr.linear_step(x, dx, alpha)
    got = want.copy()
    got[123] = np.nextafter(got[123], np.inf)
    assert gen.rel_fro(got, x + alpha * dx) <= 1e-15                      # test_linesearch's check accepts it
    assert not xr.failures(want, want) and xr.failures(got, want)


def test_bar_rejects_a_gradient_entry_missing_a_1e13_term():
    rng = np.random.default_rng(13)
    N, nx, nu, nc, nct, nc0 = 3, 4, 2, 2, 1, 4
    r = lambda *s: rng.standard_normal(s)
    g = dict(lx=r(N, nx), lu=r(N, nu), lx_N=r(nx), Jx=r(N, nx, nx), Ju=r(N, nx, nu), cJx=r(N, nc, nx), cJu=r(N, nc, nu),
             cJx_N=r(nct, nx), G0=r(nc0, nx), lam0=r(nc0), lams=r(N, nx), vs=r(N, nc), vsT=r(nct))
    g["Jx"][1, 0, 2] = 1e-13 / g["lams"][1, 0]            # one term of Lxs[1][2] is 1e-13
    Lxs, _ = pin.lagrangian_gradient(list(g["lx"]), list(g["lu"]), g["lx_N"], list(g["Jx"]), list(g["Ju"]),
                                     list(g["cJx"]), list(g["cJu"]), g["cJx_N"], g["G0"], [g["lam0"]] + list(g["lams"]),
                                     list(g["vs"]) + [g["vsT"]])
    want = np.array(Lxs)
    got = want.copy()
    got[1, 2] -= 1e-13
    assert np.max(np.abs(got - want)) <= 1e-13 * max(1.0, np.max(np.abs(want)))   # test_proxddp_inner's check
    wx, _ = xr.lagrangian_gradient(g)
    assert not xr.failures(want, wx) and xr.failures(got, wx)


def test_bar_rejects_the_neighbours_alpha_on_an_instance_boundary():
    """linear_step_v with alpha_b[j / per] off by one at the first element of instance b + 1."""
    rng = np.random.default_rng(14)
    B, per = 8, 60
    x, dx = rng.standard_normal((B, per)), rng.standard_normal((B, per))
    alpha = 0.37 * (1 + 2.0 ** -46 * np.arange(B))          # neighbouring instances' alphas are close
    want = np.stack([xr.linear_step(x[b], dx[b], alpha[b]) for b in range(B)])
    got = want.copy()
    got[4, 0] = xr.linear_step(x[4, :1], dx[4, :1], alpha[3])[0]
    assert got[4, 0] != want[4, 0]
    assert gen.rel_fro(got, x + alpha[:, None] * dx) <= 1e-15
    assert xr.failures(got, want)


def test_fddp_reference_satisfies_the_recursion():
    """Quu k = -Qu, Quu K = -Qux, Quuks = Quu k, evaluated in extended precision on the reference's own Vxx, Vx."""
    rng = np.random.default_rng(0)
    N, nx, nu, preg = 5, 4, 2, 1e-3
    d, _ = fddp_case("plain", rng, 1, N, nx, nu)
    r = hp.fddp_backward_pass(*fddp_args(d, 0), preg)
    pr = hp.MP.mpf(preg)
    for i in range(N):
        J = np.hstack([hp.mpa(d["Jx"][0, i]), hp.mpa(d["Ju"][0, i])])
        S = hp.mpa(d["Lxu"][0, i])
        hess = np.block([[hp.mpa(d["Lxx"][0, i]), S], [S.T, hp.mpa(d["Luu"][0, i])]]) + J.T @ r["Vxx"][i + 1] @ J
        grad = np.concatenate([hp.mpa(d["Lx"][0, i]), hp.mpa(d["Lu"][0, i])]) + J.T @ r["Vx"][i + 1]
        Quu = hess[nx:, nx:] + pr * hp.eye(nu)
        res = [Quu @ r["k"][i] + grad[nx:], (Quu @ r["K"][i] + hess[nx:, :nx]).ravel(), r["Quuks"][i] + grad[nx:]]
        for a in res:
            assert max(abs(v) for v in a) <= 1e-30
        assert all(r["Vxx"][i][p, q] == r["Vxx"][i][q, p] for p in range(nx) for q in range(nx))


@pytest.mark.parametrize("shape", [(12, 6, 6), (6, 3, 5), (4, 2, 1)])
def test_fddp_oracle_within_64u_of_the_reference(shape):
    nx, nu, N = shape
    rng = np.random.default_rng(nx)
    d, preg = fddp_case("plain", rng, 1, N, nx, nu)
    ref = hp.fddp_backward_pass(*fddp_args(d, 0), preg)
    got = of.backward_pass(*fddp_args(d, 0), preg)
    e = hp.fddp_errors([got], [ref])
    assert all(v <= 64 * hp.U for v in e.values()), e
