"""ab2_gar_factor_adjoint on the CPU.  The numpy restatement of the reverse step (lq_factor_adjoint_ref.py) against
torch.autograd through an independent float64 CPU torch restatement of the backward recursion, and against central
differences of that recursion; and the device program itself, compiled for the host and run on emulated lanes
(tests/emu/factor_adjoint_emu.cpp), against the restatement."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import emu_harness
import gen
import lq_adjoint_ref as aref
import lq_factor_adjoint_ref as ref
from emu_harness import run_factor_adjoint
from lq_cases import FACTOR_CASES, FACTOR_IDS, block_errors, case_records, factor_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
FAMS = ("ff", "fb", "vxx", "vx", "fft", "fbt")


def _restate(stage, term, case, mu, cot, fac):
    return ref.factor_adjoint(stage, term, fac["ff"], fac["fb"], fac["vxx"], fac["vx"], fac["fft"], fac["fbt"], cot,
                              case, mu)


@pytest.mark.parametrize("case", FACTOR_CASES, ids=FACTOR_IDS)
def test_restatement_matches_autograd(case):
    stage, term, _, _ = case_records(case, 31)
    cot = ref.random_cot(np.random.default_rng(3), case, 2)
    fac, want = ref.autograd(stage, term, case, 1e-3, cot)
    got = _restate(stage, term, case, 1e-3, cot, fac)
    errs = block_errors(got, want, case)
    assert max(errs.values()) <= 1e-12, errs
    assert not got["G0"].any() and not got["g0"].any()


@pytest.mark.parametrize("case", [(4, 2, 2, 2, 4, 5), (6, 3, 0, 2, 6, 3), (12, 6, 0, 3, 12, 2)],
                         ids=["c3_nct2", "c1_nct2", "c2_nct3"])
def test_restatement_at_small_mu(case):
    mu = 1e-8
    stage, term, _, _ = case_records(case, 32)
    cot = ref.random_cot(np.random.default_rng(4), case, 2)
    fac, want = ref.autograd(stage, term, case, mu, cot)
    errs = block_errors(_restate(stage, term, case, mu, cot, fac), want, case)
    assert max(errs.values()) <= max(1e-10, 2.4e-16 / mu), errs


@pytest.mark.parametrize("case", [FACTOR_CASES[0], FACTOR_CASES[4], FACTOR_CASES[1], FACTOR_CASES[7]], ids=[FACTOR_IDS[0], FACTOR_IDS[4], FACTOR_IDS[1], FACTOR_IDS[7]])
def test_restatement_matches_finite_differences(case):
    nx, nu, nc, nct, nc0, N = case
    mu = 1e-2
    stage, term, _, _ = case_records(case, 33)
    rng = np.random.default_rng(5)
    cot = ref.random_cot(rng, case, 2)
    so, _ = aref.stage_offsets(nx, nu, nc)
    to, _ = aref.term_offsets(nx, nct)
    ds, dt = rng.standard_normal(stage.shape), rng.standard_normal(term.shape)

    def symmetrise(x, off, k):
        M = x[..., off[0]:off[1]].reshape(*x.shape[:-1], k, k)
        x[..., off[0]:off[1]] = (0.5 * (M + np.swapaxes(M, -1, -2))).reshape(*x.shape[:-1], k * k)

    symmetrise(ds, so["Q"], nx)
    symmetrise(ds, so["R"], nu)
    symmetrise(dt, to["Q"], nx)
    fac = {k: v.numpy() for k, v in ref.torch_factor(torch.tensor(stage), torch.tensor(term), case, mu).items()}
    g = _restate(stage, term, case, mu, cot, fac)
    pairing = lambda o: sum(float((o[k].numpy() * cot[k]).sum()) for k in FAMS)
    h = 1e-6
    plus = pairing(ref.torch_factor(torch.tensor(stage + h * ds), torch.tensor(term + h * dt), case, mu))
    minus = pairing(ref.torch_factor(torch.tensor(stage - h * ds), torch.tensor(term - h * dt), case, mu))
    fd = (plus - minus) / (2 * h)
    an = float((g["stage"] * ds).sum() + (g["term"] * dt).sum())
    assert abs(fd - an) <= 1e-6 * max(abs(an), 1.0), (fd, an)


@pytest.mark.parametrize("case", FACTOR_CASES, ids=FACTOR_IDS)
def test_emulation_matches_restatement(case):
    recs = case_records(case, 34)
    mu = 1e-3
    fac = factor_oracle(recs, case, mu)
    cot = ref.random_cot(np.random.default_rng(6), case, 2)
    want = _restate(recs[0], recs[1], case, mu, cot, fac)
    for lanes, packed, head in ((32, True, 0), (7, False, 2)):
        got = run_factor_adjoint(recs, fac, cot, case, mu, lanes, packed, head)
        errs = block_errors(got, want, case)
        assert not errs or max(errs.values()) <= 1e-12, (lanes, packed, errs)
        assert not got["G0"].any() and not got["g0"].any()


def test_emulation_bit_equal_across_lanes_and_null_fields():
    case = (4, 2, 2, 2, 2, 5)
    recs = case_records(case, 35)
    fac = factor_oracle(recs, case, 1e-3)
    cot = ref.random_cot(np.random.default_rng(7), case, 2)
    base = run_factor_adjoint(recs, fac, cot, case, 1e-3, 32)
    for lanes in (3, 7, 256):
        got = run_factor_adjoint(recs, fac, cot, case, 1e-3, lanes)
        for k in base:
            assert np.array_equal(got[k], base[k]), (lanes, k)
    # a NULL field is a zero cotangent; per-instance mu
    part = dict(cot, vxx=None, ff=None)
    got = run_factor_adjoint(recs, fac, part, case, np.array([1e-3, 1e-3]), 32)
    want = _restate(recs[0], recs[1], case, 1e-3, part, fac)
    assert max(block_errors(got, want, case).values()) <= 1e-12


def test_emulation_c5_bit_equal_on_a_cta():
    case = (57, 28, 0, 0, 57, 2)
    recs = case_records(case, 36, B=1)
    fac = factor_oracle(recs, case, 1e-2)
    cot = ref.random_cot(np.random.default_rng(8), case, 1)
    want = _restate(recs[0], recs[1], case, 1e-2, cot, fac)
    base = run_factor_adjoint(recs, fac, cot, case, 1e-2, 256, packed=False)
    assert max(block_errors(base, want, case).values()) <= 1e-12
    got = run_factor_adjoint(recs, fac, cot, case, 1e-2, 32, packed=False)
    for k in base:
        assert np.array_equal(got[k], base[k]), k


@pytest.mark.parametrize("mutate,case", [(gen.make_2x2_pivots, (4, 2, 2, 2, 4, 6)),
                                         (gen.make_pivoting, (6, 3, 0, 0, 6, 6))], ids=["2x2", "interchange"])
def test_emulation_forced_pivots(mutate, case):
    recs = case_records(case, 37, mutate=mutate)
    mu = 1e-3
    cot = ref.random_cot(np.random.default_rng(9), case, 2)
    fac, want = ref.autograd(recs[0], recs[1], case, mu, cot)
    got = run_factor_adjoint(recs, factor_oracle(recs, case, mu), cot, case, mu, 32)
    errs = block_errors(got, want, case)
    assert max(errs.values()) <= 1e-10, errs


def test_every_served_shape_fits_or_is_refused():
    """Every shape a plain serial handle accepts either fits one item in 227 KB of shared memory, or the call refuses
    it (ab2_gar_factor_adjoint compares the same item size with 227 KB); C1 to C5 fit."""
    from aligator_b200 import gar
    fn = C.CFUNCTYPE(C.c_int, C.c_int, C.c_int, C.c_int, C.c_int)(("ab2_gar_supported", gar.lib()))
    bad = (C.c_int * 6)()
    largest, accepted = C.c_long(), C.c_long()
    e = emu_harness.lib()
    over = e.emu_item_size_scan(e.emu_factor_adjoint_item_bytes, 0, C.cast(fn, C.c_void_p), 130, bad,
                                C.byref(largest), C.byref(accepted))
    assert accepted.value > over >= 0
    assert 0 < largest.value <= 227 * 1024
    for nx, nu, nc in ((6, 3, 0), (12, 6, 0), (4, 2, 2), (14, 7, 0), (57, 28, 0)):
        assert e.emu_factor_adjoint_item_bytes(nx, nu, nc, 0, 0, 0, 1) <= 227 * 1024, (nx, nu, nc)
