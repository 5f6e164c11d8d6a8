"""The host emulation of the sweep programs (tests/emu/, one shared library) and the one way the CPU suite runs it.

The library compiles riccati_group.cuh, riccati_block.cuh and riccati_dense.cuh with g++: a group is G std::threads, a
CTA 32*W, sync() a std::barrier, mma.sync a fragment exchange, a TMA copy a memcpy.  `SweepParams` below mirrors
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

HERE = os.path.dirname(os.path.abspath(__file__))
EMU_DIR = os.path.join(HERE, "emu")
CSRC = os.path.join(HERE, "..", "aligator_b200", "csrc")
# built outside the source tree (which may be read-only), one copy per user and checkout
LIB = os.path.join(tempfile.gettempdir(), "ab2_emu_%d_%s" % (os.getuid(), hashlib.sha256(EMU_DIR.encode()).hexdigest()[:12]),
                   "libsweep_emu.so")
_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)


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
