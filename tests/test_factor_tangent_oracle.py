"""ab2_gar_factor_tangent on the CPU.  The numpy restatement of the tangent recursion (lq_factor_tangent_ref.py) against
torch.func.jvp through the independent float64 CPU torch restatement of the backward recursion
(test_factor_adjoint_oracle.torch_factor), against central differences of that recursion, and against the existing
reverse mode by duality; and the device program itself, compiled for the host and run on emulated lanes
(tests/emu/factor_tangent_emu.cpp), against the restatement."""
import ctypes as C
import functools
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import gen
import lq_adjoint_ref as aref
import lq_factor_adjoint_ref as adj
import lq_factor_tangent_ref as ref
from test_factor_adjoint_oracle import CASES, IDS, _oracle, _pack_vxx, _records, torch_factor

HERE = os.path.dirname(os.path.abspath(__file__))
FAMS = ("ff", "fb", "vxx", "vx", "fft", "fbt")


def random_dot(rng, case, B):
    """Tangent records with every entry random: Q, R and Q_N asymmetric, the pad double too."""
    nx, nu, nc, nct, nc0, N = case
    _, srec = aref.stage_offsets(nx, nu, nc)
    _, trec = aref.term_offsets(nx, nct)
    return dict(stage=rng.standard_normal((B, N, srec)), term=rng.standard_normal((B, trec)))


def _jvp(stage, term, case, mu, dot):
    """(factorisation, its tangent) by torch.func.jvp through torch_factor."""
    f = lambda s, t: torch_factor(s, t, case, mu)
    fac, tan = torch.func.jvp(f, (torch.tensor(stage), torch.tensor(term)),
                              (torch.tensor(dot["stage"]), torch.tensor(dot["term"])))
    return {k: v.numpy() for k, v in fac.items()}, {k: v.numpy() for k, v in tan.items()}


def _restate(stage, term, case, mu, dot, fac):
    return ref.factor_tangent(stage, term, fac["ff"], fac["fb"], fac["vxx"], fac["vx"], fac["fft"], fac["fbt"], dot,
                              case, mu)


def family_errors(got, want):
    """Relative Frobenius error of every output family of nonzero size."""
    errs = {}
    for k in FAMS:
        w = np.asarray(want[k])
        if w.size:
            e = gen.rel_fro(got[k], w)
            errs[k] = e if np.isfinite(e) else np.inf  # an entry left unwritten fails
    return errs


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_restatement_matches_jvp(case):
    stage, term, _, _ = _records(case, 51)
    dot = random_dot(np.random.default_rng(11), case, 2)
    fac, want = _jvp(stage, term, case, 1e-3, dot)
    errs = family_errors(_restate(stage, term, case, 1e-3, dot, fac), want)
    assert max(errs.values()) <= 1e-12, errs


@pytest.mark.parametrize("case", [(4, 2, 2, 2, 4, 5), (6, 3, 0, 2, 6, 3), (12, 6, 0, 3, 12, 2)],
                         ids=["c3_nct2", "c1_nct2", "c2_nct3"])
def test_restatement_at_small_mu(case):
    mu = 1e-8
    stage, term, _, _ = _records(case, 52)
    dot = random_dot(np.random.default_rng(12), case, 2)
    fac, want = _jvp(stage, term, case, mu, dot)
    errs = family_errors(_restate(stage, term, case, mu, dot, fac), want)
    assert max(errs.values()) <= max(1e-10, 2.4e-16 / mu), errs


@pytest.mark.parametrize("case", [CASES[0], CASES[4], CASES[1], CASES[7]], ids=[IDS[0], IDS[4], IDS[1], IDS[7]])
def test_restatement_matches_finite_differences(case):
    mu = 1e-2
    stage, term, _, _ = _records(case, 53)
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


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_duality_with_factor_adjoint(case):
    """<cbar, ydot> = <factor_adjoint(cbar), pdot>, with asymmetric Qd, Rd and Qd_N."""
    stage, term, _, _ = _records(case, 54)
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


# ---- host emulation of the device program ----
@functools.lru_cache(maxsize=None)
def _emu():
    src = os.path.join(HERE, "emu", "factor_tangent_emu.cpp")
    hdrs = [os.path.join(HERE, "..", "aligator_b200", "csrc", f)
            for f in ("lq_factor_tangent.cuh", "lq_resolve.cuh", "vxx_layout.h")]
    tag = hashlib.sha256(b"".join(open(p, "rb").read() for p in [src] + hdrs)).hexdigest()[:16]
    lib = os.path.join(tempfile.gettempdir(), "ab2_factor_tangent_emu_%d_%s.so" % (os.getuid(), tag))
    if not os.path.exists(lib):
        fd, tmp = tempfile.mkstemp(suffix=".so")
        os.close(fd)
        subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++20", "-fPIC", "-shared", "-pthread", "-w", "-o", tmp,
                               src])
        os.replace(tmp, lib)
    h = C.CDLL(lib)
    h.emu_factor_tangent.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
    h.emu_factor_tangent_size_scan.restype = C.c_long
    h.emu_factor_tangent_size_scan.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    h.emu_factor_tangent_item_bytes.restype = C.c_long
    h.emu_factor_tangent_item_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    return h


def out_shapes(case, B):
    nx, nu, nc, nct, nc0, N = case
    nr = nu + nc + nx
    return dict(ff=(B, N, nr), fb=(B, N, nr, nx), vxx=(B, N + 1, nx, nx), vx=(B, N + 1, nx), fft=(B, nct),
                fbt=(B, nct, nx))


def from_device(out):
    """Device-layout tangents -> the restatement's shapes: vxx blocks back from column-major."""
    return {k: (np.swapaxes(v, -1, -2) if k == "vxx" and v is not None else v) for k, v in out.items()}


def run_emu(recs, fac, dot, case, mu, lanes, packed=True, head=0, want=FAMS):
    nx, nu, nc, nct, nc0, N = case
    stage, term, _, _ = recs
    B = term.shape[0]
    head = head % N if N else 0
    if head:
        stage = np.roll(stage, head, axis=1)  # knot t in slot (t + head) mod N
    Vxx = np.asarray(fac["vxx"])
    V, V0 = _pack_vxx(Vxx) if packed else (np.ascontiguousarray(np.swapaxes(Vxx, -1, -2)), None)
    keep = [np.ascontiguousarray(a, dtype=np.float64) for a in (stage, term, fac["fb"], fac["fbt"], V)] + [V0] + \
           [np.ascontiguousarray(fac[k], dtype=np.float64) for k in ("ff", "vx", "fft")] + \
           [None if dot.get(k) is None else np.ascontiguousarray(dot[k], dtype=np.float64) for k in ("stage", "term")]
    out = {k: np.full(s, np.nan) for k, s in out_shapes(case, B).items()}
    ptr = lambda a: None if a is None or a.size == 0 else a.ctypes.data
    ins = (C.c_void_p * 11)(*[ptr(a) for a in keep])
    outs = (C.c_void_p * 6)(*[ptr(out[k]) if k in want else None for k in FAMS])
    _, srec = aref.stage_offsets(nx, nu, nc)
    dims = np.array([B, N, nx, nu, nc, nct, nc0, srec, term.shape[1], head, lanes], dtype=np.int32)
    mub = None if np.ndim(mu) == 0 else np.ascontiguousarray(mu, dtype=np.float64)
    _emu().emu_factor_tangent(dims.ctypes.data, float(mu) if mub is None else 0.0, ptr(mub), ins, outs)
    return from_device(out)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_emulation_matches_restatement(case):
    recs = _records(case, 55)
    mu = 1e-3
    fac = _oracle(recs, case, mu)
    dot = random_dot(np.random.default_rng(15), case, 2)
    want = _restate(recs[0], recs[1], case, mu, dot, fac)
    for lanes, packed, head in ((32, True, 0), (7, False, 2)):
        got = run_emu(recs, fac, dot, case, mu, lanes, packed, head)
        errs = family_errors(got, want)
        assert max(errs.values()) <= 1e-12, (lanes, packed, errs)
        assert np.array_equal(got["vxx"], np.swapaxes(got["vxx"], -1, -2))  # exactly symmetric


def test_emulation_bit_equal_across_lanes_and_null_fields():
    case = (4, 2, 2, 2, 2, 5)
    recs = _records(case, 56)
    fac = _oracle(recs, case, 1e-3)
    dot = random_dot(np.random.default_rng(16), case, 2)
    base = run_emu(recs, fac, dot, case, 1e-3, 32)
    for lanes in (3, 7, 256):
        got = run_emu(recs, fac, dot, case, 1e-3, lanes)
        for k in base:
            assert np.array_equal(got[k], base[k]), (lanes, k)
    # a NULL tangent field is zero (stage only, term only); per-instance mu
    for part in (dict(stage=dot["stage"]), dict(term=dot["term"])):
        got = run_emu(recs, fac, part, case, np.array([1e-3, 1e-3]), 32)
        want = _restate(recs[0], recs[1], case, 1e-3, part, fac)
        assert max(family_errors(got, want).values()) <= 1e-12, list(part)
    # a NULL out field is not written, and the others do not change
    got = run_emu(recs, fac, dot, case, 1e-3, 32, want=("fb", "vx"))
    for k in FAMS:
        if k in ("fb", "vx"):
            assert np.array_equal(got[k], base[k]), k
        else:
            assert np.isnan(got[k]).all(), k


def test_emulation_c5_bit_equal_on_a_cta():
    case = (57, 28, 0, 0, 57, 2)
    recs = _records(case, 57, B=1)
    fac = _oracle(recs, case, 1e-2)
    dot = random_dot(np.random.default_rng(17), case, 1)
    want = _restate(recs[0], recs[1], case, 1e-2, dot, fac)
    base = run_emu(recs, fac, dot, case, 1e-2, 256, packed=False)
    assert max(family_errors(base, want).values()) <= 1e-12
    got = run_emu(recs, fac, dot, case, 1e-2, 32, packed=False)
    for k in base:
        assert np.array_equal(got[k], base[k]), k


@pytest.mark.parametrize("mutate,case", [(gen.make_2x2_pivots, (4, 2, 2, 2, 4, 6)),
                                         (gen.make_pivoting, (6, 3, 0, 0, 6, 6))], ids=["2x2", "interchange"])
def test_emulation_forced_pivots(mutate, case):
    recs = _records(case, 58, mutate=mutate)
    mu = 1e-3
    dot = random_dot(np.random.default_rng(18), case, 2)
    _, want = _jvp(recs[0], recs[1], case, mu, dot)
    got = run_emu(recs, _oracle(recs, case, mu), dot, case, mu, 32)
    errs = family_errors(got, want)
    assert max(errs.values()) <= 1e-10, errs


def test_every_served_shape_fits_or_is_refused():
    """Every shape a plain serial handle accepts either fits one item in 227 KB of shared memory, or the call refuses
    it (ab2_gar_factor_tangent compares the same item size with 227 KB); C1 to C5 fit."""
    from aligator_b200 import gar
    fn = C.CFUNCTYPE(C.c_int, C.c_int, C.c_int, C.c_int, C.c_int)(("ab2_gar_supported", gar.lib()))
    bad = (C.c_int * 4)()
    largest, accepted = C.c_long(), C.c_long()
    e = _emu()
    over = e.emu_factor_tangent_size_scan(C.cast(fn, C.c_void_p), 130, bad, C.byref(largest), C.byref(accepted))
    assert accepted.value > over >= 0
    assert 0 < largest.value <= 227 * 1024
    for nx, nu, nc in ((6, 3, 0), (12, 6, 0), (4, 2, 2), (14, 7, 0), (57, 28, 0)):
        assert e.emu_factor_tangent_item_bytes(nx, nu, nc) <= 227 * 1024, (nx, nu, nc)
