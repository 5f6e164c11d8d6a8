"""ab2_gar_factor_tangent on the CPU.  The numpy restatement of the tangent recursion (lq_factor_tangent_ref.py) against
torch.func.jvp through the independent float64 CPU torch restatement of the backward recursion
(lq_factor_adjoint_ref.torch_factor), against central differences of that recursion, and against the existing
reverse mode by duality; and the device program itself, compiled for the host and run on emulated lanes
(tests/emu/factor_tangent_emu.cpp), against the restatement."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import emu_harness
import gen
import lq_factor_adjoint_ref as adj
import lq_factor_tangent_ref as ref
from emu_harness import run_factor_tangent
from lq_cases import FACTOR_CASES, FACTOR_IDS, case_records, factor_oracle, family_errors, random_dot
from lq_factor_adjoint_ref import torch_factor

HERE = os.path.dirname(os.path.abspath(__file__))
FAMS = ("ff", "fb", "vxx", "vx", "fft", "fbt")


def _restate(stage, term, case, mu, dot, fac):
    return ref.factor_tangent(stage, term, fac["ff"], fac["fb"], fac["vxx"], fac["vx"], fac["fft"], fac["fbt"], dot,
                              case, mu)


@pytest.mark.parametrize("case", FACTOR_CASES, ids=FACTOR_IDS)
def test_restatement_matches_jvp(case):
    stage, term, _, _ = case_records(case, 51)
    dot = random_dot(np.random.default_rng(11), case, 2)
    fac, want = ref.jvp(stage, term, case, 1e-3, dot)
    errs = family_errors(_restate(stage, term, case, 1e-3, dot, fac), want)
    assert max(errs.values()) <= 1e-12, errs


@pytest.mark.parametrize("case", [(4, 2, 2, 2, 4, 5), (6, 3, 0, 2, 6, 3), (12, 6, 0, 3, 12, 2)],
                         ids=["c3_nct2", "c1_nct2", "c2_nct3"])
def test_restatement_at_small_mu(case):
    mu = 1e-8
    stage, term, _, _ = case_records(case, 52)
    dot = random_dot(np.random.default_rng(12), case, 2)
    fac, want = ref.jvp(stage, term, case, mu, dot)
    errs = family_errors(_restate(stage, term, case, mu, dot, fac), want)
    assert max(errs.values()) <= max(1e-10, 2.4e-16 / mu), errs


@pytest.mark.parametrize("case", [FACTOR_CASES[0], FACTOR_CASES[4], FACTOR_CASES[1], FACTOR_CASES[7]], ids=[FACTOR_IDS[0], FACTOR_IDS[4], FACTOR_IDS[1], FACTOR_IDS[7]])
def test_restatement_matches_finite_differences(case):
    mu = 1e-2
    stage, term, _, _ = case_records(case, 53)
    rng = np.random.default_rng(13)
    dot = random_dot(rng, case, 2)
    cot = adj.random_cot(rng, case, 2)
    fac = {k: v.numpy() for k, v in torch_factor(torch.tensor(stage), torch.tensor(term), case, mu).items()}
    tan = _restate(stage, term, case, mu, dot, fac)
    pairing = lambda o: sum(float((np.asarray(o[k]) * cot[k]).sum()) for k in FAMS)
    h = 1e-6
    plus = pairing({k: v.numpy() for k, v in torch_factor(torch.tensor(stage + h * dot["stage"]),
                                                          torch.tensor(term + h * dot["term"]), case, mu).items()})
    minus = pairing({k: v.numpy() for k, v in torch_factor(torch.tensor(stage - h * dot["stage"]),
                                                           torch.tensor(term - h * dot["term"]), case, mu).items()})
    fd = (plus - minus) / (2 * h)
    an = pairing(tan)
    assert abs(fd - an) <= 1e-6 * max(abs(an), 1.0), (fd, an)


@pytest.mark.parametrize("case", FACTOR_CASES, ids=FACTOR_IDS)
def test_duality_with_factor_adjoint(case):
    """<cbar, ydot> = <factor_adjoint(cbar), pdot>, with asymmetric Qd, Rd and Qd_N."""
    stage, term, _, _ = case_records(case, 54)
    rng = np.random.default_rng(14)
    mu = 1e-3
    fac = {k: v.numpy() for k, v in torch_factor(torch.tensor(stage), torch.tensor(term), case, mu).items()}
    for _ in range(3):
        dot = random_dot(rng, case, 2)
        cot = adj.random_cot(rng, case, 2)
        tan = _restate(stage, term, case, mu, dot, fac)
        g = adj.factor_adjoint(stage, term, fac["ff"], fac["fb"], fac["vxx"], fac["vx"], fac["fft"], fac["fbt"], cot,
                               case, mu)
        lhs = sum(float((tan[k] * cot[k]).sum()) for k in FAMS)
        rhs = float((g["stage"] * dot["stage"]).sum() + (g["term"] * dot["term"]).sum())
        assert abs(lhs - rhs) <= 1e-12 * max(abs(lhs), 1.0), (lhs, rhs)


@pytest.mark.parametrize("case", FACTOR_CASES, ids=FACTOR_IDS)
def test_emulation_matches_restatement(case):
    recs = case_records(case, 55)
    mu = 1e-3
    fac = factor_oracle(recs, case, mu)
    dot = random_dot(np.random.default_rng(15), case, 2)
    want = _restate(recs[0], recs[1], case, mu, dot, fac)
    for lanes, packed, head in ((32, True, 0), (7, False, 2)):
        got = run_factor_tangent(recs, fac, dot, case, mu, lanes, packed, head)
        errs = family_errors(got, want)
        assert max(errs.values()) <= 1e-12, (lanes, packed, errs)
        assert np.array_equal(got["vxx"], np.swapaxes(got["vxx"], -1, -2))  # exactly symmetric


def test_emulation_bit_equal_across_lanes_and_null_fields():
    case = (4, 2, 2, 2, 2, 5)
    recs = case_records(case, 56)
    fac = factor_oracle(recs, case, 1e-3)
    dot = random_dot(np.random.default_rng(16), case, 2)
    base = run_factor_tangent(recs, fac, dot, case, 1e-3, 32)
    for lanes in (3, 7, 256):
        got = run_factor_tangent(recs, fac, dot, case, 1e-3, lanes)
        for k in base:
            assert np.array_equal(got[k], base[k]), (lanes, k)
    # a NULL tangent field is zero (stage only, term only); per-instance mu
    for part in (dict(stage=dot["stage"]), dict(term=dot["term"])):
        got = run_factor_tangent(recs, fac, part, case, np.array([1e-3, 1e-3]), 32)
        want = _restate(recs[0], recs[1], case, 1e-3, part, fac)
        assert max(family_errors(got, want).values()) <= 1e-12, list(part)
    # a NULL out field is not written, and the others do not change
    got = run_factor_tangent(recs, fac, dot, case, 1e-3, 32, want=("fb", "vx"))
    for k in FAMS:
        if k in ("fb", "vx"):
            assert np.array_equal(got[k], base[k]), k
        else:
            assert np.isnan(got[k]).all(), k


def test_emulation_c5_bit_equal_on_a_cta():
    case = (57, 28, 0, 0, 57, 2)
    recs = case_records(case, 57, B=1)
    fac = factor_oracle(recs, case, 1e-2)
    dot = random_dot(np.random.default_rng(17), case, 1)
    want = _restate(recs[0], recs[1], case, 1e-2, dot, fac)
    base = run_factor_tangent(recs, fac, dot, case, 1e-2, 256, packed=False)
    assert max(family_errors(base, want).values()) <= 1e-12
    got = run_factor_tangent(recs, fac, dot, case, 1e-2, 32, packed=False)
    for k in base:
        assert np.array_equal(got[k], base[k]), k


@pytest.mark.parametrize("mutate,case", [(gen.make_2x2_pivots, (4, 2, 2, 2, 4, 6)),
                                         (gen.make_pivoting, (6, 3, 0, 0, 6, 6))], ids=["2x2", "interchange"])
def test_emulation_forced_pivots(mutate, case):
    recs = case_records(case, 58, mutate=mutate)
    mu = 1e-3
    dot = random_dot(np.random.default_rng(18), case, 2)
    _, want = ref.jvp(recs[0], recs[1], case, mu, dot)
    got = run_factor_tangent(recs, factor_oracle(recs, case, mu), dot, case, mu, 32)
    errs = family_errors(got, want)
    assert max(errs.values()) <= 1e-10, errs


def test_every_served_shape_fits_or_is_refused():
    """Every shape a plain serial handle accepts either fits one item in 227 KB of shared memory, or the call refuses
    it (ab2_gar_factor_tangent compares the same item size with 227 KB); C1 to C5 fit."""
    from aligator_b200 import gar
    fn = C.CFUNCTYPE(C.c_int, C.c_int, C.c_int, C.c_int, C.c_int)(("ab2_gar_supported", gar.lib()))
    bad = (C.c_int * 6)()
    largest, accepted = C.c_long(), C.c_long()
    e = emu_harness.lib()
    over = e.emu_item_size_scan(e.emu_factor_tangent_item_bytes, 0, C.cast(fn, C.c_void_p), 130, bad,
                                C.byref(largest), C.byref(accepted))
    assert accepted.value > over >= 0
    assert 0 < largest.value <= 227 * 1024
    for nx, nu, nc in ((6, 3, 0), (12, 6, 0), (4, 2, 2), (14, 7, 0), (57, 28, 0)):
        assert e.emu_factor_tangent_item_bytes(nx, nu, nc, 0, 0, 0, 1) <= 227 * 1024, (nx, nu, nc)
