"""The host emulation of the theta-derivative programs of parametric problems (aligator_b200/csrc/lq_theta.cuh), built
from tests/emu/theta_emu.cpp into a library of its own, and the one way the CPU suite runs them.  The factors they
read come from the emulated parametric sweep (emu_harness.emulate('parametric', ...)), in the device layouts."""
import ctypes as C
import functools
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "theta_emu.cpp")
CSRC = os.path.join(HERE, "..", "aligator_b200", "csrc")
# built outside the source tree (which may be read-only), one copy per user and checkout
LIB = os.path.join(tempfile.gettempdir(), "ab2_emu_%d_%s" % (os.getuid(), hashlib.sha256(SRC.encode()).hexdigest()[:12]),
                   "libtheta_emu.so")
SOL = ("xs", "us", "vs", "vsT", "lam0", "lams")


def _sources():
    return [SRC, os.path.join(HERE, "emu", "item_emu.h"), os.path.join(CSRC, "lq_theta.cuh")]


@functools.lru_cache(maxsize=None)
def lib():
    """The library, rebuilt when it is older than any of its sources."""
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(s) for s in _sources()):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        # built under a temporary name and renamed into place: a concurrent test process never loads half a library
        fd, tmp = tempfile.mkstemp(suffix=".so", dir=os.path.dirname(LIB))
        os.close(fd)
        try:
            subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++20", "-fPIC", "-shared", "-pthread", "-w",
                                   "-o", tmp, SRC])
            os.replace(tmp, LIB)
        finally:
            if os.path.exists(tmp):
                os.remove(tmp)
    h = C.CDLL(LIB)
    h.emu_theta.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    h.emu_theta_item_bytes.restype = h.emu_theta_size_scan.restype = C.c_long
    h.emu_theta_item_bytes.argtypes = [C.c_int] * 7
    h.emu_theta_size_scan.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return h


def shapes(d7, B):
    """Per-direction shapes of the solution's fields; d7 = (nx, nu, nc, nct, nc0, nth, N)."""
    nx, nu, nc, nct, nc0, nth, N = d7
    return dict(xs=(B, N + 1, nx), us=(B, N, nu), vs=(B, N, nc), vsT=(B, nct), lam0=(B, nc0), lams=(B, N, nx))


def run_theta(raw, d7, lanes, chunk, dtheta=None, cot=None):
    """Run the ab2_gar_theta_tangent program (dtheta [nrhs][B][nth] given) or the ab2_gar_theta_adjoint program (cot:
    dict of [nrhs][B][...] cotangents, missing = zero) on the factors `raw` of an emulated parametric sweep (device
    layouts), `chunk` directions per item on `lanes` emulated lanes.  -> dict of the solution's fields [nrhs][B][...],
    or theta_bar [nrhs][B][nth]."""
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
