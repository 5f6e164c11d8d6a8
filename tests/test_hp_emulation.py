"""Every sweep program, executed on the CPU through the host emulation, against the extended-precision restatement of
the sweep (tests/hp_reference.py), with a tolerance set by each problem's conditioning: a program may be at most 16
times worse than the fp64 oracle on the same inputs, family by family (K, k, Z, z, Ahat, a, Vxx, vx, xs, us, vs,
lambda), or within 64 u where the oracle itself is better than that.  Also: initial conditions G0 x0 + g0 = 0 with a
dense G0 and any number of rows, homogeneous problems (exactly zero solution), and exact per-instance rescaling.

The 1e-10 comparisons of the other modules stay; these tests sit below them."""
import functools

import numpy as np
import pytest

import gen
import hp_reference as hp
from emu_harness import emulate, lib
from lq_cases import families, run_solver


# name: ((nx, nu, nc, nct, N), batch, mueq, problem transform, well conditioned)
CASES = {
    "c2": ((12, 6, 0, 0, 10), 2, 1e-8, None, True),
    "c1": ((6, 3, 0, 0, 16), 2, 1e-8, None, True),
    "c3_mu1e-3": ((4, 2, 2, 0, 20), 3, 1e-3, None, False),
    "c3_mu1e-8": ((4, 2, 2, 0, 30), 3, 1e-8, None, False),
    "c3_mu1e-11": ((4, 2, 2, 0, 30), 3, 1e-11, None, False),
    "nct": ((4, 2, 2, 3, 10), 2, 1e-3, None, False),
    "pivots_2x2": ((4, 2, 2, 0, 10), 2, 1e-3, gen.make_2x2_pivots, False),
    "interchanges": ((12, 6, 0, 0, 8), 2, 1e-8, gen.make_pivoting, False),
    "cta_7_3_0": ((7, 3, 0, 0, 8), 2, 1e-8, None, True),
    "cta_9_5_3": ((9, 5, 3, 0, 6), 2, 1e-3, None, False),
}
for _nx, _dims, _mu in ((4, (4, 2, 2, 2, 8), 1e-3), (12, (12, 6, 0, 0, 6), 1e-8)):
    for _nc0 in sorted({0, 1, _nx // 2, _nx}):
        CASES["G0_%d_nc0_%d" % (_nx, _nc0)] = (_dims, 2, _mu, ("G0", _nc0), False)


def make_problems(name):
    dims, B, mueq, transform, _ = CASES[name]
    nx, nu, nc, nct, N = dims
    probs = gen.generate_batch(1000 + sum(map(ord, name)), B, N, nx, nu, nc, nct)
    if isinstance(transform, tuple):
        gen.general_initial_condition(probs, transform[1], 77)
    elif transform is not None:
        transform(probs)
    return probs


@functools.lru_cache(maxsize=None)
def case(name):
    """(problems, extended-precision outputs rounded to fp64, oracle outputs, oracle error families)."""
    dims, B, mueq, _, _ = CASES[name]
    nx, nu, nc, nct, N = dims
    probs = make_problems(name)
    ref, _ = hp.solve(probs, mueq)
    ora = run_solver(probs, dims, mueq)
    return probs, ref, ora, hp.error_families(ora, ref, nu, nc, N)


@functools.lru_cache(maxsize=None)
def oracle_errors(name, algorithm):
    """Error families of the oracle for a program running `algorithm` ('serial', 'dense', 'legs2', 'legs3').  For the
    dense and leg programs: the larger of the serial solver's error and that of the oracle's restatement of the same
    algorithm -- both are correct fp64 solvers of the problem, and where a quantity comes out of a cancellation (a
    small z on an active row at mu = 1e-11) one of them alone can land unrepresentatively close."""
    dims, B, mueq, _, _ = CASES[name]
    probs, ref, ora, e = case(name)
    if algorithm == "serial":
        return e
    own = hp.error_families(run_solver(probs, dims, mueq, algorithm), ref, dims[1], dims[2], dims[4])
    return {f: max(v, e[f]) for f, v in own.items()}


def expand_packed(out, nx, N):
    """[B][N+1][nx*nx] column-major blocks from the packed lower triangles (slot 0 from the full Vxx0)."""
    pk, B = out["Vxx"], out["Vxx"].shape[0]
    full = np.empty((B, N + 1, nx * nx))
    full[:, 0] = out["Vxx0"]
    for t in range(1, N + 1):
        for j in range(nx):
            for i in range(nx):
                a, b = max(i, j), min(i, j)
                full[:, t, i + j * nx] = pk[:, t, b * nx - b * (b - 1) // 2 + (a - b)]
    return full


def run_program(prog, probs, dims, mueq):
    """One emulated program -> outputs in the oracle's shapes ([b, t, i, j] Vxx, zero-size arrays where empty)."""
    kind, arg, packed, legs = prog
    nx, nu, nc, nct, N = dims
    B, nc0 = len(probs), probs[0].nc0
    o = emulate(kind, probs, dims, mueq, arg, packed=packed, legs=legs)
    assert np.all(o["status"] == 0), (prog, o["status"])
    if packed:
        o["Vxx"] = expand_packed(o, nx, N)
    o["Vxx"] = o["Vxx"].reshape(B, N + 1, nx, nx).transpose(0, 1, 3, 2)
    for k, s in dict(us=(B, N, nu), vs=(B, N, nc), fbT=(B, nct, nx), ffT=(B, nct), vsT=(B, nct), lbd0=(B, nc0)).items():
        o[k] = o[k].reshape(s) if np.prod(s) else np.zeros(s)
    return o


def programs(dims, nc0):
    """(kind, arg, packed, legs) of every emulated program that runs these dimensions."""
    nx, nu, nc, nct, N = dims
    progs = []
    if lib().emu_stage_record(nx, nu, nc) > 0 and nx + nc0 <= (8 if nx <= 4 else 16 if nx <= 8 else 32):
        modes = (0, 1, 2, 3) if (nc == 0 and nx % 2 == 0 and nx >= 10) else (0, 1)
        progs += [("group", m, pk, 0) for m in modes for pk in (False, True)]
    progs.append(("block", 1, False, 0))
    if (nx, nu, nc) in ((7, 3, 0), (9, 5, 3)) and nc0 == nx:
        progs.append(("static", 1, False, 0))
    progs.append(("dense", 1, False, 0))
    if N >= 4:
        progs += [("legs", 1, False, 2), ("legs", 1, False, 3)]
    return progs


def algorithm(prog):
    """The oracle's restatement of the algorithm a program runs: the bar is that implementation's own error."""
    return {"dense": "dense", "legs": "legs%d" % prog[3]}.get(prog[0], "serial")


def prog_id(p):
    return "%s%d%s%s" % (p[0], p[1], "_packed" if p[2] else "", "_legs%d" % p[3] if p[3] else "")


ITEMS = [(n, p) for n in CASES for p in programs(CASES[n][0], make_problems(n)[0].nc0)]


@pytest.mark.parametrize("name,prog", ITEMS, ids=["%s-%s" % (n, prog_id(p)) for n, p in ITEMS])
def test_program_against_extended_precision(name, prog):
    dims, B, mueq, _, _ = CASES[name]
    nx, nu, nc, nct, N = dims
    probs, ref, ora, _ = case(name)
    got = run_program(prog, probs, dims, mueq)
    e_oracle = oracle_errors(name, algorithm(prog))
    e_kernel = hp.error_families(got, ref, nu, nc, N, families(prog))
    bad = hp.violations(e_kernel, e_oracle)
    assert not bad, hp.table("%s %s" % (name, prog_id(prog)), e_oracle, e_kernel)


@pytest.mark.parametrize("name", [n for n in CASES if CASES[n][4]])
def test_oracle_meets_the_floor_on_well_conditioned_cases(name):
    """The oracle's own numerics are pinned, not only its agreement with the kernels: every family within 64 u of the
    extended-precision result."""
    probs, ref, ora, e_oracle = case(name)
    assert max(e_oracle.values()) <= hp.FLOOR, e_oracle


@pytest.mark.parametrize("name", ["c1", "G0_12_nc0_6"])
def test_reference_solves_the_whole_problem(name):
    """The extended-precision solution satisfies the whole-problem KKT system (gen.lqr_dense_kkt) to ~1e-30, and its
    gains, Vxx and vx satisfy the stage equations that define them."""
    dims, B, mueq, _, _ = CASES[name]
    probs = make_problems(name)[:1]
    _, hps = hp.solve(probs, mueq)
    assert hp.kkt_residual(probs[0], mueq, hps[0]) <= 1e-30
    assert hp.stage_equation_residual(probs[0], mueq, hps[0]) <= 1e-30
    # and its fp64 rounding agrees with an independent fp64 dense solve of the whole problem
    xs, us, vs, lb = gen.lqr_dense_solve(probs[0], mueq)
    assert gen.rel_fro(np.concatenate(xs), hp.to64(np.concatenate(list(hps[0]["xs"])))) <= 1e-12


@pytest.mark.parametrize("name", [n for n in CASES if CASES[n][4]])
def test_tolerance_rejects_a_1e12_error_that_1e10_accepts(name):
    """One entry of one knot's K, and separately one entry of Vxx, off by a relative 1e-12 in otherwise correct
    outputs: the conditioning-aware tolerance rejects it, the flat 1e-10 relative Frobenius comparison does not."""
    dims, B, mueq, _, _ = CASES[name]
    nx, nu, nc, nct, N = dims
    probs, ref, ora, e_oracle = case(name)
    prog = programs(dims, probs[0].nc0)[0]
    good = run_program(prog, probs, dims, mueq)
    assert not hp.violations(hp.error_families(good, ref, nu, nc, N), e_oracle)
    t = N // 2
    for fam, key, sl in (("K", "fb", np.s_[0, t, :nu]), ("Vxx", "Vxx", np.s_[0, t])):
        bad = {k: np.array(v, copy=True) for k, v in good.items()}
        blk = bad[key][sl]
        i = np.unravel_index(np.argmax(np.abs(blk)), blk.shape)
        blk[i] *= 1 + 1e-12
        assert not np.array_equal(bad[key], good[key])
        assert gen.rel_fro(bad[key][sl], ora[key][sl]) <= 1e-10  # the old comparison accepts it
        assert fam in hp.violations(hp.error_families(bad, ref, nu, nc, N), e_oracle), fam


# ---------------------------------------------------------------------------------------------------------------------
# Homogeneous problems and exact rescaling
# ---------------------------------------------------------------------------------------------------------------------
ZERO_KEYS = ("ff", "ffT", "xs", "us", "vs", "vsT", "lbd0", "lbdas")


@pytest.mark.parametrize("dims,nc0", [((4, 2, 2, 2, 6), 2), ((12, 6, 0, 0, 5), 12), ((7, 3, 0, 0, 5), 3),
                                      ((9, 5, 3, 2, 4), 9)])
def test_homogeneous_problem_has_exactly_zero_solution(dims, nc0):
    """q = r = f = d = g0 = 0: every feedforward, the trajectory and the multipliers are exactly zero in every
    program -- a stray read of uninitialised memory would show."""
    nx, nu, nc, nct, N = dims
    probs = gen.generate_batch(61, 3, N, nx, nu, nc, nct)
    if nc0 != nx:
        gen.general_initial_condition(probs, nc0, 3)
    gen.make_homogeneous(probs)
    for prog in programs(dims, nc0):
        got = run_program(prog, probs, dims, 1e-3 if nc + nct else 1e-8)
        for k in ZERO_KEYS:
            assert np.all(got[k] == 0.0), (prog, k)
        assert np.all(np.isfinite(got["fb"])) and np.any(got["fb"] != 0), prog


EXACT = ("ff", "fb", "ffT", "fbT", "xs", "us", "vs", "vsT", "lbd0", "kkt0")
SCALED = ("Vxx", "vx", "lbdas", "Vxx0")
EXPONENTS = (-60, 0, 37, 60, -23)


def check_rescaling(run, probs, mueq):
    """Instance b scaled by c_b = 2**EXPONENTS[b] through the per-instance mu: every output bit for bit that of the
    unscaled instance (Vxx, vx, lbdas: c_b times it)."""
    B = len(probs)
    base = run(probs, np.full(B, mueq))
    scaled, mu_b = gen.scale_instances(probs, EXPONENTS[:B], mueq)
    got = run(scaled, mu_b)
    c = 2.0 ** np.array(EXPONENTS[:B], dtype=np.float64)
    for k in EXACT + SCALED:
        if k not in base:
            continue
        want = base[k] * c.reshape((B,) + (1,) * (base[k].ndim - 1)) if k in SCALED else base[k]
        assert np.array_equal(got[k], want, equal_nan=True), k


@pytest.mark.parametrize("dims,nc0", [((4, 2, 2, 2, 6), 2), ((12, 6, 0, 0, 5), 6), ((9, 5, 3, 0, 4), 9),
                                      ((7, 3, 0, 2, 4), 7)])
def test_exact_per_instance_rescaling(dims, nc0):
    """Every KKT matrix of instance b is exactly c_b times the original: same pivots, same rounding.  Catches an
    absolute threshold anywhere in the sweep and any leak between the instances of a batch.  Not for leg mode, whose
    condensed refinement stops at an absolute threshold, nor for the dense program: its stage system holds the
    dynamics rows [B 0 0 -I] (not scaled) beside the cost rows (scaled by c_b), so it is not c_b times the original
    and its pivots and rounding legitimately change (measured: K differs by ~1e-15 relative at c = 2, ~1e-11 at
    c = 2^-60, the oracle's restatement of the dense algorithm alike)."""
    nx, nu, nc, nct, N = dims
    probs = gen.generate_batch(71, 5, N, nx, nu, nc, nct)
    if nc0 != nx:
        gen.general_initial_condition(probs, nc0, 4)
    for prog in programs(dims, nc0):
        if prog[0] in ("legs", "dense"):
            continue
        kind, arg, packed, _ = prog
        run = lambda ps, mu: {k: v for k, v in emulate(kind, ps, dims, mu, arg, packed=packed).items()
                              if k not in ("status", "pivstat")}
        check_rescaling(run, probs, 1e-3 if nc + nct else 1e-8)
