"""ab2_gar_factor_adjoint on the CPU.  The numpy restatement of the reverse step (lq_factor_adjoint_ref.py) against
torch.autograd through an independent float64 CPU torch restatement of the backward recursion, and against central
differences of that recursion; and the device program itself, compiled for the host and run on emulated lanes
(tests/emu/factor_adjoint_emu.cpp), against the restatement."""
import ctypes as C
import functools
import os

import numpy as np
import pytest
import torch

import emu_harness
import gen
import lq_adjoint_ref as aref
import lq_factor_adjoint_ref as ref
from oracle import gar_oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
FAMS = ("ff", "fb", "vxx", "vx", "fft", "fbt")

# (nx, nu, nc, nct, nc0, N): C1, C2 and C3 dims, nc > 0, nct > 0, horizon 0 and 1
CASES = [(6, 3, 0, 0, 6, 4), (6, 3, 0, 2, 3, 1), (12, 6, 0, 0, 12, 3), (12, 6, 0, 3, 1, 0), (4, 2, 2, 2, 4, 5),
         (4, 2, 2, 0, 0, 1), (4, 2, 2, 2, 2, 0), (5, 2, 1, 1, 0, 3)]
IDS = ["nx%d_nu%d_nc%d_nct%d_nc0%d_N%d" % c for c in CASES]


def _records(case, seed, B=2, mutate=None):
    nx, nu, nc, nct, nc0, N = case
    probs = gen.general_initial_condition(gen.generate_batch(seed, B, N, nx, nu, nc, nct), nc0, seed)
    if mutate:
        probs = mutate(probs) or probs
    _, srec = aref.stage_offsets(nx, nu, nc)
    stage = np.zeros((B, N, srec))
    for b, p in enumerate(probs):
        for t in range(N):
            r = gen.stage_record(p.stages[t])
            stage[b, t, :r.size] = r
    term = np.stack([gen.term_record(p.stages[N]) for p in probs])
    G0 = np.stack([np.asarray(p.G0).ravel(order="F") for p in probs]).reshape(B, nc0 * nx)
    g0 = np.stack([np.asarray(p.g0) for p in probs]).reshape(B, nc0)
    return stage, term, G0, g0


def torch_factor(stage, term, case, mu):
    """The backward recursion in float64 CPU torch: (ff, fb, vxx, vx, fft, fbt) in the restatement's shapes.  Stage
    KKT systems by torch.linalg.solve, Q and R as (P + P^T) / 2 of the stored blocks."""
    nx, nu, nc, nct, nc0, N = case
    B = term.shape[0]
    so, _ = aref.stage_offsets(nx, nu, nc)
    to, _ = aref.term_offsets(nx, nct)
    blk = lambda rec, off, m, n: rec[..., off[0]:off[1]].reshape(*rec.shape[:-1], n, m).transpose(-1, -2)
    sym = lambda P: 0.5 * (P + P.transpose(-1, -2))
    T = lambda M: M.transpose(-1, -2)
    mv = lambda M, x: (M @ x[..., None])[..., 0]
    QN, qN = sym(blk(term, to["Q"], nx, nx)), term[:, to["q"][0]:to["q"][1]]
    CN, dN = blk(term, to["C"], nct, nx), term[:, to["d"][0]:to["d"][1]]
    fbt, fft = CN / mu, dN / mu
    V = QN + T(CN) @ fbt
    v = qN + mv(T(CN), fft)
    Vs, vs, ffs, fbs = [V], [v], [], []
    for t in range(N - 1, -1, -1):
        r = stage[:, t]
        A, Bm, f = blk(r, so["A"], nx, nx), blk(r, so["B"], nx, nu), r[:, so["f"][0]:so["f"][1]]
        Q, S, R = sym(blk(r, so["Q"], nx, nx)), blk(r, so["S"], nx, nu), sym(blk(r, so["R"], nu, nu))
        q, rr = r[:, so["q"][0]:so["q"][1]], r[:, so["r"][0]:so["r"][1]]
        Cm, D, d = blk(r, so["C"], nc, nx), blk(r, so["D"], nc, nu), r[:, so["d"][0]:so["d"][1]]
        vplus = v + mv(V, f)
        Sh, Qh = S + T(A) @ V @ Bm, Q + T(A) @ V @ A
        top = torch.cat([R + T(Bm) @ V @ Bm, T(D)], -1)
        bot = torch.cat([D, -mu * torch.eye(nc, dtype=torch.float64).expand(B, nc, nc)], -1)
        M = torch.cat([top, bot], -2)
        Y = torch.cat([torch.cat([T(Sh), (rr + mv(T(Bm), vplus))[..., None]], -1),
                       torch.cat([Cm, d[..., None]], -1)], -2)
        X = -torch.linalg.solve(M, Y)
        K, k, Z, z = X[:, :nu, :nx], X[:, :nu, nx], X[:, nu:, :nx], X[:, nu:, nx]
        fbs.append(torch.cat([K, Z, A + Bm @ K], -2))
        ffs.append(torch.cat([k, z, f + mv(Bm, k)], -1))
        V = Qh + Sh @ K + T(Cm) @ Z
        v = q + mv(T(A), vplus) + mv(Sh, k) + mv(T(Cm), z)
        Vs.append(V)
        vs.append(v)
    st = lambda xs, shape: torch.stack(xs[::-1], 1) if xs else torch.zeros(shape, dtype=torch.float64)
    nr = nu + nc + nx
    return dict(ff=st(ffs, (B, 0, nr)), fb=st(fbs, (B, 0, nr, nx)), vxx=torch.stack(Vs[::-1], 1),
                vx=torch.stack(vs[::-1], 1), fft=fft, fbt=fbt)


def _autograd(stage, term, case, mu, cot):
    s = torch.tensor(stage, requires_grad=True)
    t = torch.tensor(term, requires_grad=True)
    out = torch_factor(s, t, case, mu)
    loss = sum((out[k] * torch.tensor(cot[k])).sum() for k in FAMS)
    gs, gt = torch.autograd.grad(loss, (s, t), allow_unused=True)
    zero = lambda g, x: np.zeros(x.shape) if g is None else g.numpy()
    return {k: v.detach().numpy() for k, v in out.items()}, dict(stage=zero(gs, stage), term=zero(gt, term))


def _restate(stage, term, case, mu, cot, fac):
    return ref.factor_adjoint(stage, term, fac["ff"], fac["fb"], fac["vxx"], fac["vx"], fac["fft"], fac["fbt"], cot,
                              case, mu)


def block_errors(got, want, case):
    """Relative Frobenius error of every record block (gradient family) of the stage and terminal records."""
    nx, nu, nc, nct, nc0, N = case
    so, _ = aref.stage_offsets(nx, nu, nc)
    to, _ = aref.term_offsets(nx, nct)
    errs = {}
    for name, off, key in [(k, v, "stage") for k, v in so.items()] + [("N" + k, v, "term") for k, v in to.items()]:
        w = want[key][..., off[0]:off[1]]
        if w.size:
            e = gen.rel_fro(got[key][..., off[0]:off[1]], w)
            errs[name] = e if np.isfinite(e) else np.inf  # an entry left unwritten fails
    return errs


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_restatement_matches_autograd(case):
    stage, term, _, _ = _records(case, 31)
    cot = ref.random_cot(np.random.default_rng(3), case, 2)
    fac, want = _autograd(stage, term, case, 1e-3, cot)
    got = _restate(stage, term, case, 1e-3, cot, fac)
    errs = block_errors(got, want, case)
    assert max(errs.values()) <= 1e-12, errs
    assert not got["G0"].any() and not got["g0"].any()


@pytest.mark.parametrize("case", [(4, 2, 2, 2, 4, 5), (6, 3, 0, 2, 6, 3), (12, 6, 0, 3, 12, 2)],
                         ids=["c3_nct2", "c1_nct2", "c2_nct3"])
def test_restatement_at_small_mu(case):
    mu = 1e-8
    stage, term, _, _ = _records(case, 32)
    cot = ref.random_cot(np.random.default_rng(4), case, 2)
    fac, want = _autograd(stage, term, case, mu, cot)
    errs = block_errors(_restate(stage, term, case, mu, cot, fac), want, case)
    assert max(errs.values()) <= max(1e-10, 2.4e-16 / mu), errs


@pytest.mark.parametrize("case", [CASES[0], CASES[4], CASES[1], CASES[7]], ids=[IDS[0], IDS[4], IDS[1], IDS[7]])
def test_restatement_matches_finite_differences(case):
    nx, nu, nc, nct, nc0, N = case
    mu = 1e-2
    stage, term, _, _ = _records(case, 33)
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
    fac = {k: v.numpy() for k, v in torch_factor(torch.tensor(stage), torch.tensor(term), case, mu).items()}
    g = _restate(stage, term, case, mu, cot, fac)
    pairing = lambda o: sum(float((o[k].numpy() * cot[k]).sum()) for k in FAMS)
    h = 1e-6
    plus = pairing(torch_factor(torch.tensor(stage + h * ds), torch.tensor(term + h * dt), case, mu))
    minus = pairing(torch_factor(torch.tensor(stage - h * ds), torch.tensor(term - h * dt), case, mu))
    fd = (plus - minus) / (2 * h)
    an = float((g["stage"] * ds).sum() + (g["term"] * dt).sum())
    assert abs(fd - an) <= 1e-6 * max(abs(an), 1.0), (fd, an)


# ---- host emulation of the device program ----
@functools.lru_cache(maxsize=None)
def _emu():
    h = emu_harness.lib()
    h.emu_factor_adjoint.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
    h.emu_factor_adjoint_size_scan.restype = C.c_long
    h.emu_factor_adjoint_size_scan.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    h.emu_factor_adjoint_item_bytes.restype = C.c_long
    h.emu_factor_adjoint_item_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    return h


def _pack_vxx(Vxx):
    """[B][N+1][nx][nx] (row index first) -> the packed layout of vxx_layout.h."""
    B, K, nx, _ = Vxx.shape
    P = (nx * (nx + 1) // 2 + 1) & ~1
    pk = np.zeros((B, K, P))
    for j in range(nx):
        c0 = j * nx - j * (j - 1) // 2
        pk[:, :, c0:c0 + nx - j] = Vxx[:, :, j:, j]
    return pk, np.ascontiguousarray(np.swapaxes(Vxx[:, 0], -1, -2)).reshape(B, nx * nx)


def _oracle(recs, case, mu):
    nx, nu, nc, nct, nc0, N = case
    B = recs[1].shape[0]
    bo = orc.BatchedOracle(nx, nu, nc, nct, nc0, N, B, *[np.ascontiguousarray(a) for a in recs])
    bo.sweep(mu, nthreads=1)
    assert np.all(bo.status == 1)
    o = bo.get()
    return dict(ff=o["ff"], fb=o["fb"], vxx=o["Vxx"], vx=o["vx"], fft=o["ffT"], fbt=o["fbT"])


def device_cot(cot, case, B):
    """Restatement-shaped cotangents -> the device layouts (vxx column-major per block); None stays None."""
    out = {}
    for k, v in cot.items():
        if v is None:
            out[k] = None
        elif k == "vxx":
            out[k] = np.ascontiguousarray(np.swapaxes(v, -1, -2))
        else:
            out[k] = np.ascontiguousarray(v)
    return out


def run_emu(recs, fac, cot, case, mu, lanes, packed=True, head=0):
    nx, nu, nc, nct, nc0, N = case
    stage, term, _, _ = recs
    B = term.shape[0]
    head = head % N if N else 0
    if head:
        stage = np.roll(stage, head, axis=1)  # knot t in slot (t + head) mod N
    Vxx = np.asarray(fac["vxx"])
    V, V0 = _pack_vxx(Vxx) if packed else (np.ascontiguousarray(np.swapaxes(Vxx, -1, -2)), None)
    dc = device_cot(cot, case, B)
    keep = [np.ascontiguousarray(a, dtype=np.float64) for a in
            (stage, term, fac["fb"], fac["fbt"], V)] + [V0] + \
           [np.ascontiguousarray(fac[k], dtype=np.float64) for k in ("ff", "vx", "fft")] + [dc.get(k) for k in FAMS]
    _, srec = aref.stage_offsets(nx, nu, nc)
    out = dict(stage=np.full((B, N, srec), np.nan), term=np.full(term.shape, np.nan), G0=np.full((B, nc0 * nx), np.nan),
               g0=np.full((B, nc0), np.nan))
    ptr = lambda a: None if a is None or a.size == 0 else a.ctypes.data
    ins = (C.c_void_p * 15)(*[ptr(a) for a in keep])
    outs = (C.c_void_p * 4)(*[ptr(out[k]) for k in ("stage", "term", "G0", "g0")])
    dims = np.array([B, N, nx, nu, nc, nct, nc0, srec, term.shape[1], head, lanes], dtype=np.int32)
    mub = None if np.ndim(mu) == 0 else np.ascontiguousarray(mu, dtype=np.float64)
    _emu().emu_factor_adjoint(dims.ctypes.data, float(mu) if mub is None else 0.0, ptr(mub), ins, outs)
    return out


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_emulation_matches_restatement(case):
    recs = _records(case, 34)
    mu = 1e-3
    fac = _oracle(recs, case, mu)
    cot = ref.random_cot(np.random.default_rng(6), case, 2)
    want = _restate(recs[0], recs[1], case, mu, cot, fac)
    for lanes, packed, head in ((32, True, 0), (7, False, 2)):
        got = run_emu(recs, fac, cot, case, mu, lanes, packed, head)
        errs = block_errors(got, want, case)
        assert not errs or max(errs.values()) <= 1e-12, (lanes, packed, errs)
        assert not got["G0"].any() and not got["g0"].any()


def test_emulation_bit_equal_across_lanes_and_null_fields():
    case = (4, 2, 2, 2, 2, 5)
    recs = _records(case, 35)
    fac = _oracle(recs, case, 1e-3)
    cot = ref.random_cot(np.random.default_rng(7), case, 2)
    base = run_emu(recs, fac, cot, case, 1e-3, 32)
    for lanes in (3, 7, 256):
        got = run_emu(recs, fac, cot, case, 1e-3, lanes)
        for k in base:
            assert np.array_equal(got[k], base[k]), (lanes, k)
    # a NULL field is a zero cotangent; per-instance mu
    part = dict(cot, vxx=None, ff=None)
    got = run_emu(recs, fac, part, case, np.array([1e-3, 1e-3]), 32)
    want = _restate(recs[0], recs[1], case, 1e-3, part, fac)
    assert max(block_errors(got, want, case).values()) <= 1e-12


def test_emulation_c5_bit_equal_on_a_cta():
    case = (57, 28, 0, 0, 57, 2)
    recs = _records(case, 36, B=1)
    fac = _oracle(recs, case, 1e-2)
    cot = ref.random_cot(np.random.default_rng(8), case, 1)
    want = _restate(recs[0], recs[1], case, 1e-2, cot, fac)
    base = run_emu(recs, fac, cot, case, 1e-2, 256, packed=False)
    assert max(block_errors(base, want, case).values()) <= 1e-12
    got = run_emu(recs, fac, cot, case, 1e-2, 32, packed=False)
    for k in base:
        assert np.array_equal(got[k], base[k]), k


@pytest.mark.parametrize("mutate,case", [(gen.make_2x2_pivots, (4, 2, 2, 2, 4, 6)),
                                         (gen.make_pivoting, (6, 3, 0, 0, 6, 6))], ids=["2x2", "interchange"])
def test_emulation_forced_pivots(mutate, case):
    recs = _records(case, 37, mutate=mutate)
    mu = 1e-3
    cot = ref.random_cot(np.random.default_rng(9), case, 2)
    fac, want = _autograd(recs[0], recs[1], case, mu, cot)
    got = run_emu(recs, _oracle(recs, case, mu), cot, case, mu, 32)
    errs = block_errors(got, want, case)
    assert max(errs.values()) <= 1e-10, errs


def test_every_served_shape_fits_or_is_refused():
    """Every shape a plain serial handle accepts either fits one item in 227 KB of shared memory, or the call refuses
    it (ab2_gar_factor_adjoint compares the same item size with 227 KB); C1 to C5 fit."""
    from aligator_b200 import gar
    fn = C.CFUNCTYPE(C.c_int, C.c_int, C.c_int, C.c_int, C.c_int)(("ab2_gar_supported", gar.lib()))
    bad = (C.c_int * 4)()
    largest, accepted = C.c_long(), C.c_long()
    e = _emu()
    over = e.emu_factor_adjoint_size_scan(C.cast(fn, C.c_void_p), 130, bad, C.byref(largest), C.byref(accepted))
    assert accepted.value > over >= 0
    assert 0 < largest.value <= 227 * 1024
    for nx, nu, nc in ((6, 3, 0), (12, 6, 0), (4, 2, 2), (14, 7, 0), (57, 28, 0)):
        assert e.emu_factor_adjoint_item_bytes(nx, nu, nc) <= 227 * 1024, (nx, nu, nc)
