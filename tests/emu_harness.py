"""The host emulation of the sweep programs and the per-item programs (tests/emu/, one shared library) and the one way
the CPU suite runs them.

The library compiles riccati_group.cuh, riccati_block.cuh and riccati_dense.cuh with g++: a group is G std::threads, a
CTA 32*W, sync() a std::barrier, mma.sync a fragment exchange, a TMA copy a memcpy.  The item programs (lq_resolve.cuh,
lq_theta.cuh, lq_factor_adjoint.cuh, lq_factor_tangent.cuh) run the same way, one item after another.  `SweepParams` below mirrors
ab2::SweepParams field for field; the library checks the mirror when it loads."""
import ctypes as C
import functools
import glob
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import gen
import lq_adjoint_ref
import lq_cases
import lq_factor_adjoint_ref
import lq_resolve_ref
from oracle import gar_oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
EMU_DIR = os.path.join(HERE, "emu")
CSRC = os.path.join(HERE, "..", "aligator_b200", "csrc")
# built outside the source tree (which may be read-only), one copy per user and checkout
LIB = os.path.join(tempfile.gettempdir(), "ab2_emu_%d_%s" % (os.getuid(), hashlib.sha256(EMU_DIR.encode()).hexdigest()[:12]),
                   "libsweep_emu.so")
_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)
SOL = lq_resolve_ref.SOL  # the fields of a solution, as resolve and the theta tangent write them


class SweepParams(C.Structure):
    _fields_ = [("N", C.c_int), ("nct", C.c_int), ("nc0", C.c_int), ("batch", C.c_int),
                ("mueq", C.c_double), ("do_bwd", C.c_int), ("do_fwd", C.c_int)] + \
               [(n, _dp) for n in ("stage", "term", "G0", "g0", "ff", "fb", "Vxx", "vx", "ffT",
                                   "fbT", "kkt0", "xs", "us", "vs", "vsT", "lbd0", "lbdas")] + \
               [("status", _ip), ("pivstat", _ip), ("stagger_ns", C.c_int), ("num_sms", C.c_int),
                ("ctas_per_sm", C.c_int), ("stage_head", C.c_int), ("nth", C.c_int)] + \
               [(n, _dp) for n in ("theta", "fth", "Vxt", "Vtt", "vt", "kkt0fth", "thGrad", "thHess")] + \
               [("legs", C.c_int), ("clk", C.c_void_p), ("cond", _dp),
                ("peer_world", C.c_int), ("peer_dst", C.c_void_p * 8), ("peer_off", C.c_longlong),
                ("Vxx0", _dp), ("mueq_b", _dp)]


def layout_mismatches(lib, mirror=SweepParams):
    """What differs between a ctypes mirror and the library's ab2::SweepParams: size, then every field's offset."""
    bad = []
    if C.sizeof(mirror) != lib.emu_sweep_params_size():
        bad.append(("sizeof", C.sizeof(mirror), lib.emu_sweep_params_size()))
    for name, *_ in mirror._fields_:
        want = lib.emu_sweep_params_offset(name.encode())
        if getattr(mirror, name).offset != want:
            bad.append((name, getattr(mirror, name).offset, want))
    return bad


def _sources():
    """Everything the library is built from: every file under tests/emu/ and every header of the CUDA sources."""
    srcs = [os.path.join(EMU_DIR, f) for f in os.listdir(EMU_DIR) if os.path.isfile(os.path.join(EMU_DIR, f))]
    return srcs + glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(CSRC, "*.cuh"))


@functools.lru_cache(maxsize=None)
def lib():
    """The emulation library, rebuilt when it is older than any of its sources."""
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(s) for s in _sources()):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        # built under a temporary name and renamed into place: a concurrent test process never loads half a library
        fd, tmp = tempfile.mkstemp(suffix=".so", dir=os.path.dirname(LIB))
        os.close(fd)
        try:
            subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++20", "-fPIC", "-shared", "-pthread", "-w",
                                   "-o", tmp, os.path.join(EMU_DIR, "emu.cpp")])
            os.replace(tmp, LIB)
        finally:
            if os.path.exists(tmp):
                os.remove(tmp)
    h = C.CDLL(LIB)
    h.emu_sweep_params_offset.argtypes = [C.c_char_p]
    for name in ("emu_factor_adjoint", "emu_factor_tangent", "emu_resolve"):
        getattr(h, name).argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
    h.emu_theta.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    for name in ("emu_resolve", "emu_theta", "emu_factor_adjoint", "emu_factor_tangent"):
        getattr(h, name + "_item_bytes").restype = C.c_long
        getattr(h, name + "_item_bytes").argtypes = [C.c_int] * 7  # nx, nu, nc, nct, nc0, nth, chunk
    h.emu_item_size_scan.restype = C.c_long
    h.emu_item_size_scan.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    bad = layout_mismatches(h)
    assert not bad, "tests/emu_harness.py SweepParams does not match ab2::SweepParams: %s" % bad
    return h


def _F(a):
    return np.asarray(a, dtype=np.float64).ravel(order="F")


def _parametric_records(probs, N):
    """Stage / terminal records of parametric problems: the plain record followed by Gx, Gu, Gv, Gth, gamma, each
    block at its offset in the tests' mirror of the record layout."""
    def record(k, off):
        rec = np.zeros(max(e for _, e in off.values()))
        for name, (s, e) in off.items():
            rec[s:e] = _F(getattr(k, name))
        return rec

    rows = lambda *ms: (np.shape(m)[0] for m in ms)
    stage = []
    for p in probs:
        recs = [record(k, lq_adjoint_ref.stage_offsets(*rows(k.Q, k.R, k.C, k.Gth))[0]) for k in p.stages[:N]]
        stage.append(np.stack(recs) if recs else np.zeros((0, 0)))
    term = np.stack([record(k, lq_adjoint_ref.term_offsets(*rows(k.Q, k.C, k.Gth))[0]) for k in (p.stages[N] for p in probs)])
    return stage, term, np.stack([_F(p.G0) for p in probs]), np.stack([np.asarray(p.g0) for p in probs])


KINDS = ("group", "block", "static", "parametric", "legs", "dense")


def emulate(kind, probs, dims, mueq, arg=0, packed=False, legs=0, collapse=False, nth=0, theta=None, peers=None):
    """Run one sweep program over the problems `probs` on the CPU and return its outputs, NaN where nothing was written.

    kind: 'group' (arg = mode: 0/1 lane-per-column step with a single / double record buffer, 2/3 tensor-core step
    with a double / single one; packed: Vxx stored as the device builds store it), 'block' (the CTA-per-instance
    program at run-time dimensions, arg = emulated warps), 'static' (its compile-time specialisation), 'parametric'
    (nth > 0 parameters, forward at `theta`), 'legs' (leg mode with `legs` legs; collapse: collapseFeedback too) or
    'dense' (the stage-dense program).  dims = (nx, nu, nc, nct, N).  mueq: a number, or a [batch] array that selects
    the per-instance mu as the *_v launches do.  peers (group): (receive buffers of every rank, offset in doubles)."""
    assert kind in KINDS, kind
    h = lib()
    nx, nu, nc, nct, N = dims
    B, nc0 = len(probs), probs[0].nc0
    if kind == "group":
        srec = h.emu_stage_record(nx, nu, nc)
    else:
        srec = h.emu_block_stage_record(nx, nu, nc, nth if kind == "parametric" else 0)
    assert srec > 0, "shape not instantiated"
    if kind == "parametric":
        rows, term, G0, g0 = _parametric_records(probs, N)
        stage = np.zeros((B, max(N, 1), srec))
        for b, r in enumerate(rows):
            stage[b, :N, :r.shape[-1]] = r
    else:
        stage, term, G0, g0 = gen.pack_problems(probs)
        if N > 0 and stage.shape[-1] != srec:
            stage = np.concatenate([stage, np.zeros(stage.shape[:-1] + (srec - stage.shape[-1],))], -1)
    nr = nu + nc + nx + (nx if kind == "dense" else 0)
    z = lambda *s: np.full(s if np.prod(s) > 0 else (1,), np.nan)
    zz = lambda *s: np.zeros(s if np.prod(s) > 0 else (1,))
    vxx = h.emu_vxx_packed_doubles(nx) if packed else nx * nx
    out = dict(ff=z(B, N, nr), fb=z(B, N, nr, nx), Vxx=z(B, N + 1, vxx), vx=z(B, N + 1, nx), ffT=z(B, nct),
               fbT=z(B, nct, nx), kkt0=z(B, nx + nc0), xs=z(B, N + 1, nx), us=z(B, N, nu), vs=z(B, N, nc),
               vsT=z(B, nct), lbd0=z(B, nc0), lbdas=z(B, N, nx))
    if packed:
        out["Vxx0"] = z(B, nx * nx)
    if kind == "legs":
        out.update(fth=zz(B, N, nr, nx), Vxt=zz(B, N + 1, nx * nx), Vtt=zz(B, N + 1, nx * nx), vt=zz(B, N + 1, nx),
                   cond=z(B, nc0 + nx * (2 * legs - 1)))
    if kind == "parametric":
        out.update(fth=z(B, N, nr, nth), Vxt=z(B, N + 1, nx * nth), Vtt=z(B, N + 1, nth * nth), vt=z(B, N + 1, nth),
                   kkt0fth=z(B, nx + nc0, nth), thGrad=z(B, nth), thHess=z(B, nth * nth))
    status, pivstat = np.full(B, -1, dtype=np.int32), np.zeros(B, dtype=np.int32)
    inputs = dict(stage=stage, term=term, G0=G0, g0=g0)
    if theta is not None:
        inputs["theta"] = theta
    scalar = np.ndim(mueq) == 0
    if not scalar:
        inputs["mueq_b"] = mueq
    inputs = {k: np.ascontiguousarray(v, dtype=np.float64) for k, v in inputs.items()}
    p = SweepParams()
    p.N, p.nct, p.nc0, p.batch, p.mueq, p.do_bwd, p.do_fwd = N, nct, nc0, B, (mueq if scalar else np.nan), 1, 1
    p.nth, p.legs = (nx, legs) if kind == "legs" else (nth, 0)
    for k, v in list(inputs.items()) + list(out.items()):
        setattr(p, k, v.ctypes.data_as(_dp))
    p.status = status.ctypes.data_as(_ip)
    p.pivstat = pivstat.ctypes.data_as(_ip)
    if peers is not None:  # sharded batch: SweepParams::peer_*
        bufs, off = peers
        p.peer_world = len(bufs)
        for w, buf in enumerate(bufs):
            p.peer_dst[w] = buf.ctypes.data
        p.peer_off = off
    if kind == "group":
        rc = h.emu_sweep(nx, nu, nc, arg, int(packed), C.byref(p))
    elif kind in ("block", "parametric"):
        rc = h.emu_block_sweep(nx, nu, nc, arg, C.byref(p))
    elif kind == "static":
        rc = h.emu_block_sweep_static(nx, nu, nc, arg, C.byref(p))
    elif kind == "legs":
        rc = h.emu_block_legs(nx, nu, nc, arg, 3 | (4 if collapse else 0), C.byref(p))
    else:
        rc = h.emu_dense_sweep(nx, nu, nc, arg, C.byref(p))
    assert rc == 0, (kind, rc)
    out["status"], out["pivstat"] = status, pivstat
    return out


def pack_vxx(Vxx):
    """[B][N+1][nx][nx] (row index first) -> the packed layout of vxx_layout.h: packed lower triangles, and the full
    column-major slot-0 blocks."""
    B, K, nx, _ = Vxx.shape
    P = (nx * (nx + 1) // 2 + 1) & ~1
    pk = np.zeros((B, K, P))
    for j in range(nx):
        c0 = j * nx - j * (j - 1) // 2
        pk[:, :, c0:c0 + nx - j] = Vxx[:, :, j:, j]
    return pk, np.ascontiguousarray(np.swapaxes(Vxx[:, 0], -1, -2)).reshape(B, nx * nx)


def from_device(out):
    """Device-layout tangents -> the restatement's shapes: vxx blocks back from column-major."""
    return {k: (np.swapaxes(v, -1, -2) if k == "vxx" and v is not None else v) for k, v in out.items()}


def run_factor_adjoint(recs, fac, cot, case, mu, lanes, packed=True, head=0):
    """Run the ab2_gar_factor_adjoint program (tests/emu/factor_adjoint_emu.cpp) on `lanes` emulated lanes per instance:
    the gradient records of the cotangent `cot` of the factorisation `fac` (the restatement\'s shapes).  packed: Vxx
    in the warp kernel\'s packed layout; head: the stage ring\'s head."""
    nx, nu, nc, nct, nc0, N = case
    stage, term, _, _ = recs
    B = term.shape[0]
    head = head % N if N else 0
    if head:
        stage = np.roll(stage, head, axis=1)  # knot t in slot (t + head) mod N
    Vxx = np.asarray(fac["vxx"])
    V, V0 = pack_vxx(Vxx) if packed else (np.ascontiguousarray(np.swapaxes(Vxx, -1, -2)), None)
    dc = lq_cases.device_cot(cot, case, B)
    keep = [np.ascontiguousarray(a, dtype=np.float64) for a in
            (stage, term, fac["fb"], fac["fbt"], V)] + [V0] + \
           [np.ascontiguousarray(fac[k], dtype=np.float64) for k in ("ff", "vx", "fft")] + [dc.get(k) for k in lq_factor_adjoint_ref.COT]
    _, srec = lq_adjoint_ref.stage_offsets(nx, nu, nc)
    out = dict(stage=np.full((B, N, srec), np.nan), term=np.full(term.shape, np.nan), G0=np.full((B, nc0 * nx), np.nan),
               g0=np.full((B, nc0), np.nan))
    ptr = lambda a: None if a is None or a.size == 0 else a.ctypes.data
    ins = (C.c_void_p * 15)(*[ptr(a) for a in keep])
    outs = (C.c_void_p * 4)(*[ptr(out[k]) for k in ("stage", "term", "G0", "g0")])
    dims = np.array([B, N, nx, nu, nc, nct, nc0, srec, term.shape[1], head, lanes], dtype=np.int32)
    mub = None if np.ndim(mu) == 0 else np.ascontiguousarray(mu, dtype=np.float64)
    lib().emu_factor_adjoint(dims.ctypes.data, float(mu) if mub is None else 0.0, ptr(mub), ins, outs)
    return out


def run_factor_tangent(recs, fac, dot, case, mu, lanes, packed=True, head=0, want=lq_factor_adjoint_ref.COT):
    """Run the ab2_gar_factor_tangent program (tests/emu/factor_tangent_emu.cpp) like run_factor_adjoint: the tangents
    of the factorisation along the record tangent `dot`, only the families in `want` written."""
    nx, nu, nc, nct, nc0, N = case
    stage, term, _, _ = recs
    B = term.shape[0]
    head = head % N if N else 0
    if head:
        stage = np.roll(stage, head, axis=1)  # knot t in slot (t + head) mod N
    Vxx = np.asarray(fac["vxx"])
    V, V0 = pack_vxx(Vxx) if packed else (np.ascontiguousarray(np.swapaxes(Vxx, -1, -2)), None)
    keep = [np.ascontiguousarray(a, dtype=np.float64) for a in (stage, term, fac["fb"], fac["fbt"], V)] + [V0] + \
           [np.ascontiguousarray(fac[k], dtype=np.float64) for k in ("ff", "vx", "fft")] + \
           [None if dot.get(k) is None else np.ascontiguousarray(dot[k], dtype=np.float64) for k in ("stage", "term")]
    out = {k: np.full(s, np.nan) for k, s in lq_cases.out_shapes(case, B).items()}
    ptr = lambda a: None if a is None or a.size == 0 else a.ctypes.data
    ins = (C.c_void_p * 11)(*[ptr(a) for a in keep])
    outs = (C.c_void_p * 6)(*[ptr(out[k]) if k in want else None for k in lq_factor_adjoint_ref.COT])
    _, srec = lq_adjoint_ref.stage_offsets(nx, nu, nc)
    dims = np.array([B, N, nx, nu, nc, nct, nc0, srec, term.shape[1], head, lanes], dtype=np.int32)
    mub = None if np.ndim(mu) == 0 else np.ascontiguousarray(mu, dtype=np.float64)
    lib().emu_factor_tangent(dims.ctypes.data, float(mu) if mub is None else 0.0, ptr(mub), ins, outs)
    return from_device(out)


def run_resolve(recs, o, h, case, nrhs, mu, lanes, chunk, packed, head):
    """Run the ab2_gar_resolve program (tests/emu/resolve_emu.cpp): the solutions of the nrhs right-hand sides h on
    the oracle\'s factorisation o, `chunk` right-hand sides per item on `lanes` emulated lanes."""
    nx, nu, nc, nct, nc0, N = case
    stage, term, G0, _ = recs
    B = term.shape[0]
    if head and N:
        stage = np.roll(stage, head, axis=1)  # knot t in slot (t + head) mod N
    Vxx = np.asarray(o["Vxx"])
    if packed:
        V, V0 = pack_vxx(Vxx)
    else:
        V, V0 = np.ascontiguousarray(np.swapaxes(Vxx, -1, -2)), None
    keep = [np.ascontiguousarray(a, dtype=np.float64) for a in (stage, term, G0, o["fb"], o["fbT"], V)]
    keep.append(None if V0 is None else np.ascontiguousarray(V0))
    hf = lq_resolve_ref.full_rhs(h, case, B, nrhs)
    keep += [np.ascontiguousarray(hf[k]) for k in lq_resolve_ref.RHS]
    out = {k: np.full((nrhs,) + s, np.nan) for k, s in zip(SOL, lq_resolve_ref.rhs_shapes(case, B).values())}
    ptr = lambda a: None if a is None or a.size == 0 else a.ctypes.data
    ins = (C.c_void_p * 13)(*[ptr(a) for a in keep])
    outs = (C.c_void_p * 6)(*[ptr(out[k]) for k in SOL])
    _, srec = lq_adjoint_ref.stage_offsets(nx, nu, nc)
    dims = np.array([B, N, nx, nu, nc, nct, nc0, srec, term.shape[1], head if N else 0, nrhs, chunk, lanes],
                    dtype=np.int32)
    mub = None if np.ndim(mu) == 0 else np.ascontiguousarray(mu, dtype=np.float64)
    lib().emu_resolve(dims.ctypes.data, float(mu) if mub is None else 0.0, ptr(mub), ins, outs)
    return out


def shapes(d7, B):
    """Per-direction shapes of the solution's fields; d7 = (nx, nu, nc, nct, nc0, nth, N)."""
    nx, nu, nc, nct, nc0, nth, N = d7
    return dict(xs=(B, N + 1, nx), us=(B, N, nu), vs=(B, N, nc), vsT=(B, nct), lam0=(B, nc0), lams=(B, N, nx))


def run_theta(raw, d7, lanes, chunk, dtheta=None, cot=None):
    """Run the ab2_gar_theta_tangent program (dtheta [nrhs][B][nth] given) or the ab2_gar_theta_adjoint program (cot:
    dict of [nrhs][B][...] cotangents, missing = zero) on the factors `raw` of an emulated parametric sweep
    (emulate('parametric', ...), device layouts), `chunk` directions per item on `lanes` emulated lanes.  -> dict of
    the solution's fields [nrhs][B][...], or theta_bar [nrhs][B][nth]."""
    nx, nu, nc, nct, nc0, nth, N = d7
    B = raw["xs"].shape[0]
    adjoint = dtheta is None
    nrhs = (next(v for v in cot.values() if v is not None).shape[0]) if adjoint else dtheta.shape[0]
    ptr = lambda a: None if a is None or a.size == 0 else a.ctypes.data
    keep = [np.ascontiguousarray(raw[k], dtype=np.float64) for k in ("fb", "fth", "fbT", "Vxx", "Vxt", "kkt0fth")]
    if adjoint:
        keep += [None if cot.get(k) is None else np.ascontiguousarray(cot[k], dtype=np.float64) for k in SOL]
        out = {"theta_bar": np.full((nrhs, B, nth), np.nan)}
    else:
        keep.append(np.ascontiguousarray(dtheta, dtype=np.float64))
        out = {k: np.full((nrhs,) + s, np.nan) for k, s in shapes(d7, B).items()}
    ins = (C.c_void_p * 12)(*[ptr(a) for a in keep] + [None] * (12 - len(keep)))
    outs = (C.c_void_p * 6)(*[ptr(a) for a in out.values()] + [None] * (6 - len(out)))
    dims = np.array([B, N, nx, nu, nc, nct, nc0, nth, nrhs, chunk, lanes, int(adjoint)], dtype=np.int32)
    lib().emu_theta(dims.ctypes.data, ins, outs)
    return out


def check_against_oracle(nx, nu, nc, nct, N, B, mueq, seed, tol=1e-10, style="conditioned", db=0,
                         pivoting=False, block=0):
    probs = gen.generate_batch(seed, B, N, nx, nu, nc, nct, style=style)
    if pivoting:
        gen.make_pivoting(probs)
    # block = 0: the warp-per-instance group program; block = NW > 0: the CTA-per-instance program of
    # riccati_block.cuh with NW emulated warps; block = -NW: its compile-time specialisation (StaticBlockDims)
    kind = "group" if block == 0 else ("block" if block > 0 else "static")
    got = emulate(kind, probs, (nx, nu, nc, nct, N), mueq, db if block == 0 else abs(block))
    got["Vxx"] = got["Vxx"].reshape(B, N + 1, nx, nx).transpose(0, 1, 3, 2)
    assert np.all(got["status"] == 0)
    stage, term, G0, g0 = gen.pack_problems(probs)
    bo = orc.BatchedOracle(nx, nu, nc, nct, probs[0].nc0, N, B, stage, term, G0, g0)
    bo.sweep(mueq, nthreads=1)
    ref = bo.get()
    worst = {}
    for b in range(B):
        for t in range(N):
            worst["K"] = max(worst.get("K", 0), gen.rel_fro(got["fb"][b, t, :nu], ref["fb"][b, t, :nu]))
            worst["k"] = max(worst.get("k", 0), gen.rel_fro(got["ff"][b, t, :nu], ref["ff"][b, t, :nu]))
            worst["fb"] = max(worst.get("fb", 0), gen.rel_fro(got["fb"][b, t], ref["fb"][b, t]))
            worst["ff"] = max(worst.get("ff", 0), gen.rel_fro(got["ff"][b, t], ref["ff"][b, t]))
        for t in range(N + 1):
            worst["Vxx"] = max(worst.get("Vxx", 0), gen.rel_fro(got["Vxx"][b, t], ref["Vxx"][b, t]))
            worst["vx"] = max(worst.get("vx", 0), gen.rel_fro(got["vx"][b, t], ref["vx"][b, t]))
        for key in ("xs", "us", "vs", "lbdas", "lbd0", "vsT"):
            if ref[key].size:
                worst[key] = max(worst.get(key, 0), gen.rel_fro(got[key][b], ref[key][b]))
    # K alone on control-constrained knots is limited by eps*cond(KKT) ~ 6e-17/mueq between
    # any two correct fp64 solvers (SURVEY Appendix C); everything else is gated at `tol`.
    tolk = max(tol, 2.4e-16 / mueq) if nc > 0 else tol
    bad = {k: v for k, v in worst.items() if not v <= (tolk if k in ("K", "k") else tol)}
    assert not bad, (bad, worst)
    # structural semantics (A1): Vxx_t symmetric for t >= 1 when N > 0
    for t in range(1, N + 1):
        assert np.array_equal(got["Vxx"][0, t], got["Vxx"][0, t].T)
    return worst
