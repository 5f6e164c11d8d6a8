"""The parametric and leg-mode sweep programs, executed on the CPU through the host emulation, against the
extended-precision restatement (tests/hp_reference.py: solve_parametric, solve_legs) at the conditioning-aware bar of
tests/test_hp_emulation.py: e_kernel <= max(16 e_oracle, 64 u) for every family, the theta families (Kth, Zth, Yth,
Vxt, Vtt, vt, kkt0fth, thGrad, thHess) and collapse_feedback's gain included.  Also exact properties: homogeneous
problems, per-instance rescaling by powers of two, the terminal knot's theta terms, and forward at theta = 0."""
import functools

import numpy as np
import pytest

import gen
import hp_reference as hp
import lq_cases
from emu_harness import emulate
from lq_cases import PARAM_CASES


def warps(nx, nu, nc, nth):
    """The fewest emulated warps the parametric program runs these dimensions on (33 theta columns: two)."""
    return (max(nx + 1, nu + nc, 2 * nx, nu + nc + nx, nth) + 31) // 32


def product_layout(o, nx, nth):
    """Raw emulated outputs -> the product's layouts (those of CudaRiccatiBatch.get)."""
    B, K = o["Vxx"].shape[:2]
    o = dict(o)
    o["Vxx"] = o["Vxx"].reshape(B, K, nx, nx).transpose(0, 1, 3, 2)
    if "Vxt" in o:
        o["Vxt"] = o["Vxt"].reshape(B, K, nth, nx).transpose(0, 1, 3, 2)
        o["Vtt"] = o["Vtt"].reshape(B, K, nth, nth).transpose(0, 1, 3, 2)
    if "thHess" in o:
        o["thHess"] = o["thHess"].reshape(B, nth, nth).transpose(0, 2, 1)
    return o


def run_parametric(probs, shape, mueq, thetas, nw=None):
    nx, nu, nc, nct, nth, N = shape
    o = emulate("parametric", probs, (nx, nu, nc, nct, N), mueq, nw or warps(nx, nu, nc, nth), nth=nth,
                theta=None if thetas is None else np.ascontiguousarray(thetas))
    assert np.all(o["status"] == 0), o["status"]
    o = product_layout(o, nx, nth)
    B, nc0 = len(probs), probs[0].nc0
    for k, s in dict(us=(B, N, nu), vs=(B, N, nc), fbT=(B, nct, nx), ffT=(B, nct), vsT=(B, nct), lbd0=(B, nc0),
                     fb=(B, N, nu + nc + nx, nx), ff=(B, N, nu + nc + nx), fth=(B, N, nu + nc + nx, nth),
                     lbdas=(B, N, nx)).items():
        o[k] = o[k].reshape(s) if np.prod(s) else np.zeros(s)
    return o


@functools.lru_cache(maxsize=None)
def param_case(name):
    """(problems, thetas, restatement fp64 outputs, oracle's error families)."""
    shape, B, mueq, _, _, _ = PARAM_CASES[name]
    probs, thetas = lq_cases.param_problems(name)
    ref, _ = hp.solve_parametric_batch(probs, mueq, thetas)
    return probs, thetas, ref, lq_cases.param_oracle_errors(probs, mueq, thetas, ref)


@pytest.mark.parametrize("name", list(PARAM_CASES))
def test_parametric_program_against_extended_precision(name):
    shape, B, mueq, _, _, _ = PARAM_CASES[name]
    nx, nu, nc, nct, nth, N = shape
    probs, thetas, ref, e_oracle = param_case(name)
    got = run_parametric(probs, shape, mueq, thetas)
    e_kernel = hp.error_families(got, ref, nu, nc, N)
    assert {"Vxt", "Vtt", "vt", "kkt0fth", "thGrad", "thHess"} <= set(e_kernel)
    print("\n" + hp.table("parametric %s" % name, e_oracle, e_kernel))
    lq_cases.check_bar(e_kernel, e_oracle, "parametric %s" % name)


@pytest.mark.parametrize("name", ["nth1", "nth_nx"])
def test_tolerance_rejects_a_1e12_error_in_theta_terms(name):
    """One entry of one knot's Vxt, and separately one entry of one knot's Kth, off by a relative 1e-12 in otherwise
    correct outputs: the bar rejects it, the flat 1e-10 relative Frobenius comparison accepts it."""
    shape, B, mueq, _, _, _ = PARAM_CASES[name]
    nx, nu, nc, nct, nth, N = shape
    probs, thetas, ref, e_oracle = param_case(name)
    good = run_parametric(probs, shape, mueq, thetas)
    assert not hp.violations(hp.error_families(good, ref, nu, nc, N), e_oracle)
    t = N // 2
    for fam, key, sl in (("Vxt", "Vxt", np.s_[0, t]), ("Kth", "fth", np.s_[0, t, :nu])):
        bad = {k: np.array(v, copy=True) for k, v in good.items()}
        blk = bad[key][sl]
        i = np.unravel_index(np.argmax(np.abs(blk)), blk.shape)
        blk[i] *= 1 + 1e-12
        assert not np.array_equal(bad[key], good[key])
        assert gen.rel_fro(bad[key][sl], good[key][sl]) <= 1e-10  # the old comparison accepts it
        assert fam in hp.violations(hp.error_families(bad, ref, nu, nc, N), e_oracle), fam


# ---------------------------------------------------------------------------------------------------------------------
# Exact properties
# ---------------------------------------------------------------------------------------------------------------------
EXACT_SHAPES = [(4, 2, 2, 2, 3, 6), (6, 3, 0, 0, 6, 5), (5, 2, 1, 0, 33, 3)]


def exact_problems(shape, seed, B=3, nc0=None):
    nx, nu, nc, nct, nth, N = shape
    probs = [lq_cases.make_problem([seed, b], N, nx, nu, nc, nct, nth, gv=True) for b in range(B)]
    if nc0 is not None:
        gen.general_initial_condition(probs, nc0, seed)
    return probs


@pytest.mark.parametrize("shape", EXACT_SHAPES)
def test_homogeneous_parametric_problem(shape):
    """q = r = f = d = g0 = 0 and gamma = 0: ff, vx, vt, thGrad, kkt0 and the theta-free rollout are exactly zero."""
    nx, nu, nc, nct, nth, N = shape
    probs = gen.make_homogeneous(exact_problems(shape, 31, nc0=nx // 2))
    for p in probs:
        for k in p.stages:
            k.gamma[...] = 0.0
    mueq = 1e-3 if nc + nct else 1e-8
    got = run_parametric(probs, shape, mueq, None)
    for k in ("ff", "vx", "vt", "thGrad", "kkt0", "xs", "us", "vs", "vsT", "lbd0", "lbdas"):
        assert np.all(got[k] == 0.0), k
    for k in ("fth", "Vxt", "Vtt", "thHess", "kkt0fth"):
        assert np.all(np.isfinite(got[k])) and np.any(got[k] != 0), k


EXPONENTS = (-60, 0, 37, 60, -23)


@pytest.mark.parametrize("shape", EXACT_SHAPES)
def test_parametric_exact_per_instance_rescaling(shape):
    """Instance b scaled by c_b = 2**s_b with mu_b = c_b mu (the parametric blocks Gx, Gu, Gv, Gth, gamma too): the
    gains, Kth, Zth, Yth, kkt0.fth and the rollout at theta bit for bit those of the unscaled instance, Vxt, Vtt, vt,
    thGrad and thHess exactly c_b times them."""
    nx, nu, nc, nct, nth, N = shape
    B = len(EXPONENTS)
    probs = exact_problems(shape, 41, B, nc0=max(nx - 1, 0))
    thetas = np.random.default_rng(41).standard_normal((B, nth))
    mueq = 1e-3 if nc + nct else 1e-8
    base = run_parametric(probs, shape, np.full(B, mueq), thetas)
    scaled, mu_b = gen.scale_instances(probs, EXPONENTS, mueq)
    got = run_parametric(scaled, shape, mu_b, thetas)
    c = 2.0 ** np.array(EXPONENTS, dtype=np.float64)
    for k in ("fb", "ff", "fth", "kkt0", "kkt0fth", "xs", "us", "vs", "lbd0"):
        assert np.array_equal(got[k], base[k]), k
    for k in ("Vxx", "vx", "Vxt", "Vtt", "vt", "thGrad", "thHess", "lbdas"):
        assert np.array_equal(got[k], base[k] * c.reshape((B,) + (1,) * (base[k].ndim - 1))), k


@pytest.mark.parametrize("shape", EXACT_SHAPES + [(4, 2, 2, 2, 3, 0)])
def test_terminal_theta_terms_and_forward_at_zero(shape):
    """The terminal knot's theta terms are the reference's copies (riccati-kernel.hxx:185-192 with nu = 0): Vxt_N = Gx_N,
    Vtt_N = Gth_N, vt_N = gamma_N bit for bit; and forward at theta = 0 is forward without theta, bit for bit."""
    nx, nu, nc, nct, nth, N = shape
    probs = exact_problems(shape, 51)
    mueq = 1e-3 if nc + nct else 1e-8
    free = run_parametric(probs, shape, mueq, None)
    zero = run_parametric(probs, shape, mueq, np.zeros((len(probs), nth)))
    for b, p in enumerate(probs):
        T = p.stages[N]
        assert np.array_equal(free["Vxt"][b, N], T.Gx) and np.array_equal(free["Vtt"][b, N], T.Gth)
        assert np.array_equal(free["vt"][b, N], T.gamma)
    for k in ("xs", "us", "vs", "vsT", "lbd0", "lbdas"):
        assert np.array_equal(free[k], zero[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# Leg mode
# ---------------------------------------------------------------------------------------------------------------------
# (nx, nu, nc, nct, nc0, N, legs, mueq)
LEG_CASES = [(4, 2, 0, 0, 4, 11, 2, 1e-8), (4, 2, 2, 0, 4, 13, 3, 1e-3), (5, 3, 2, 2, 2, 9, 4, 1e-2),
             (3, 2, 0, 0, 3, 10, 8, 1e-8), (6, 3, 1, 2, 0, 17, 3, 1e-3), (7, 3, 0, 0, 7, 14, 6, 1e-8)]


def run_legs(probs, dims, mueq, T, collapse=False):
    nx, nu, nc, nct, N = dims
    o = emulate("legs", probs, dims, mueq, 1, legs=T, collapse=collapse)
    assert np.all(o["status"] == 0), o["status"]
    o = product_layout(o, nx, nx)
    B = len(probs)
    for k, s in dict(us=(B, N, nu), vs=(B, N, nc), vsT=(B, nct), lbd0=(B, probs[0].nc0)).items():
        o[k] = o[k].reshape(s) if np.prod(s) else np.zeros(s)
    return o


@pytest.mark.parametrize("shape", LEG_CASES, ids=["nx%d_nu%d_nc%d_nct%d_nc0%d_N%d_legs%d" % s[:7] for s in LEG_CASES])
def test_legs_program_against_extended_precision(shape):
    """Every factor family of every knot of every leg (the theta terms on the knots that carry them) and
    collapse_feedback's first gain, against the leg restatement at the bar set by the oracle's ParallelRiccatiSolver."""
    nx, nu, nc, nct, nc0, N, T, mueq = shape
    probs = gen.generate_batch(400 + N + T, 2, N, nx, nu, nc, nct)
    if nc0 != nx:
        gen.general_initial_condition(probs, nc0, 14)
    dims = (nx, nu, nc, nct, N)
    ref, _ = hp.solve_legs_batch(probs, mueq, T)
    e_oracle = hp.error_families(lq_cases.oracle_legs(probs, mueq, T), ref, nu, nc, N, lq_cases.LEG_FAMILIES)
    got = run_legs(probs, dims, mueq, T)
    got["collapse"] = run_legs(probs, dims, mueq, T, collapse=True)["fb"][:, 0, :nu]
    e_kernel = hp.error_families(got, ref, nu, nc, N, lq_cases.LEG_FAMILIES)
    assert {"Kth", "Vxt", "Vtt", "vt", "collapse"} <= set(e_kernel)
    print("\n" + hp.table("legs %s" % (shape,), e_oracle, e_kernel))
    lq_cases.check_bar(e_kernel, e_oracle, "legs %s" % (shape,))
