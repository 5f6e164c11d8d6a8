"""The sweep programs with a per-instance mu (ab2::InstanceMu, what the *_v launches run), executed on the CPU through
the host emulation (tests/emu/per_instance_emu.cpp): the warp-per-instance group program with both step
implementations and both record-buffer layouts, the CTA-per-instance program, its leg mode and the stage-dense program.

Each instance's outputs must be array-equal to the scalar program run at that instance's mu; instances that share
their records but not their mu must differ where mu enters; and every instance matches the oracle at its own mu."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import gen
from oracle import gar_oracle as orc
from test_group_emulation import SweepParams, _dp
from test_group_packed_emulation import SweepParamsPacked

HERE = os.path.dirname(os.path.abspath(__file__))
EMU_DIR = os.path.join(HERE, "emu")
EMU_LIB = os.path.join(EMU_DIR, "libper_instance_emu.so")
CSRC = os.path.join(HERE, "..", "aligator_b200", "csrc")

MUS = (1.0, 1e-2, 1e-5)


def _lib():
    srcs = [os.path.join(EMU_DIR, f) for f in ("per_instance_emu.cpp", "group_packed_emu.cpp", "group_emu.cpp",
                                                "block_emu.cpp")] + \
        [os.path.join(CSRC, f) for f in ("riccati_group.cuh", "riccati_block.cuh", "riccati_dense.cuh",
                                         "riccati_configs.h", "vxx_layout.h")]
    if (not os.path.exists(EMU_LIB)
            or os.path.getmtime(EMU_LIB) < max(os.path.getmtime(s) for s in srcs)):
        subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++20", "-fPIC", "-shared", "-pthread", "-w",
                               "-o", EMU_LIB, srcs[0]])
    lib = C.CDLL(EMU_LIB)
    for f in ("emu_pi_sweep", "emu_pi_block_sweep", "emu_pi_block_legs", "emu_pi_dense_sweep"):
        getattr(lib, f).argtypes = [C.c_int] * 4 + [C.c_void_p, C.c_long, C.c_void_p]
    return lib


def run(lib, kind, probs, dims, mu, arg, legs=0):
    """kind: 'group' (arg = mode: 0/1 lane-per-column single/double buffer, 2/3 tensor-core double/single), 'block'
    (arg = emulated warps), 'legs', 'dense'.  mu: a number (the scalar program) or a [batch] array (InstanceMu)."""
    nx, nu, nc, nct, N = dims
    B, nc0 = len(probs), probs[0].nc0
    stage, term, G0, g0 = gen.pack_problems(probs)
    srec = lib.emu_stage_record(nx, nu, nc) if kind == "group" else lib.emu_block_stage_record(nx, nu, nc)
    if N > 0 and stage.shape[-1] != srec:
        stage = np.concatenate([stage, np.zeros(stage.shape[:-1] + (srec - stage.shape[-1],))], -1)
    stage = np.ascontiguousarray(stage)
    nr = nu + nc + nx + (nx if kind == "dense" else 0)
    packed = kind == "group"
    P = lib.emu_vxx_packed_doubles(nx)
    z = lambda *s: np.full(s if np.prod(s) > 0 else (1,), np.nan)
    zz = lambda *s: np.zeros(s if np.prod(s) > 0 else (1,))
    out = dict(ff=z(B, N, nr), fb=z(B, N, nr, nx), Vxx=z(B, N + 1, P if packed else nx * nx), vx=z(B, N + 1, nx),
               ffT=z(B, nct), fbT=z(B, nct, nx), kkt0=z(B, nx + nc0), xs=z(B, N + 1, nx), us=z(B, N, nu),
               vs=z(B, N, nc), vsT=z(B, nct), lbd0=z(B, nc0), lbdas=z(B, N, nx))
    if packed:
        out["Vxx0"] = z(B, nx * nx)
    if kind == "legs":
        out.update(fth=zz(B, N, nr, nx), Vxt=zz(B, N + 1, nx * nx), Vtt=zz(B, N + 1, nx * nx), vt=zz(B, N + 1, nx),
                   cond=z(B, nc0 + nx * (2 * legs - 1)))
    status, pivstat = np.full(B, -1, dtype=np.int32), np.zeros(B, dtype=np.int32)
    p = SweepParamsPacked() if packed else SweepParams()
    scalar = np.isscalar(mu)
    p.N, p.nct, p.nc0, p.batch, p.mueq, p.do_bwd, p.do_fwd = N, nct, nc0, B, (mu if scalar else np.nan), 1, 1
    if kind == "legs":
        p.nth, p.legs = nx, legs
    for k, v in dict(stage=stage, term=term, G0=G0, g0=g0, **out).items():
        setattr(p, k, v.ctypes.data_as(_dp))
    p.status = status.ctypes.data_as(C.POINTER(C.c_int))
    p.pivstat = pivstat.ctypes.data_as(C.POINTER(C.c_int))
    assert C.sizeof(p) <= lib.emu_pi_params_offset()
    if scalar:
        rc = dict(group=lambda: lib.emu_sweep_packed(nx, nu, nc, arg, C.byref(p)),
                  block=lambda: lib.emu_block_sweep(nx, nu, nc, arg, C.byref(p)),
                  legs=lambda: lib.emu_block_legs(nx, nu, nc, arg, 3, C.byref(p)),
                  dense=lambda: lib.emu_dense_sweep(nx, nu, nc, arg, C.byref(p)))[kind]()
    else:
        mu = np.ascontiguousarray(mu, dtype=np.float64)
        f = dict(group=lib.emu_pi_sweep, block=lib.emu_pi_block_sweep, legs=lib.emu_pi_block_legs,
                 dense=lib.emu_pi_dense_sweep)[kind]
        rc = f(nx, nu, nc, arg, C.addressof(p), C.sizeof(p), mu.ctypes.data)
    assert rc == 0, rc
    out["status"], out["pivstat"] = status, pivstat
    return out


def _batch(dims, seed):
    """Instances 0, 1, 2 share one problem (and get mu = 1, 1e-2, 1e-5); instance 3 is another problem."""
    nx, nu, nc, nct, N = dims
    a = gen.generate_batch(seed, 1, N, nx, nu, nc, nct)[0]
    b = gen.generate_batch(seed + 1, 1, N, nx, nu, nc, nct)[0]
    return [a, a.copy(), a.copy(), b], np.array([MUS[0], MUS[1], MUS[2], MUS[1]])


def _check(lib, kind, dims, arg, legs=0, gains=True, seed=3):
    nx, nu, nc, nct, N = dims
    probs, mu_b = _batch(dims, seed + nx)
    got = run(lib, kind, probs, dims, mu_b, arg, legs)
    want = {}
    for v in MUS:  # every instance as the scalar program at its own mu
        r = run(lib, kind, probs, dims, v, arg, legs)
        for k in r:
            if r[k].shape[0] == len(probs):  # (arrays of zero size are one-element placeholders)
                want.setdefault(k, np.empty_like(r[k]))[mu_b == v] = r[k][mu_b == v]
    for k in want:
        assert np.array_equal(got[k], want[k], equal_nan=True), (kind, k)
    assert np.all(got["status"] == 0)
    # the guard: same records, different mu -> different Z = C / mu, z = d / mu and multipliers
    for k in ("fbT", "ffT", "vsT") + (("vs",) if nc else ()):
        for i, j in ((0, 1), (1, 2), (0, 2)):
            assert not np.array_equal(got[k][i], got[k][j]), (kind, k, i, j)
    # each instance against the oracle at its own mu: the solution, and the feedback gains of the programs that compute
    # the proximal solver's (the legs' gains are parametric in the next leg's head, the dense program's are its own)
    stage, term, G0, g0 = gen.pack_problems(probs)
    for b in range(len(probs)):
        bo = orc.BatchedOracle(nx, nu, nc, nct, probs[0].nc0, N, 1, stage[b:b + 1], term[b:b + 1], G0[b:b + 1],
                               g0[b:b + 1])
        bo.sweep(mu_b[b], nthreads=1)
        ref = bo.get()
        for k in ("xs", "us", "vs", "lbdas"):
            if ref[k].size:
                assert gen.rel_fro(got[k][b], ref[k][0]) <= 1e-10, (kind, k, b, mu_b[b])
        if gains:
            assert gen.rel_fro(got["fb"][b, :, :nu], ref["fb"][0, :, :nu]) <= 1e-10, (kind, "K", b)


GROUP = [((2, 2, 2, 2, 6), m) for m in (0, 1)] + [((4, 2, 2, 2, 7), m) for m in (0, 1)] + \
    [((5, 2, 2, 2, 5), m) for m in (0, 1)] + [((12, 6, 6, 3, 4), m) for m in (0, 1)] + \
    [((12, 6, 0, 3, 5), m) for m in (2, 3)] + [((14, 7, 0, 2, 4), m) for m in (2, 3)]


@pytest.mark.parametrize("dims,mode", GROUP, ids=["%d_%d_%d_nct%d-mode%d" % (d[:4] + (m,)) for d, m in GROUP])
def test_group_program(dims, mode):
    """mode 0/1: lane-per-column step, single / double record buffer; 2/3: tensor-core step, double / single."""
    _check(_lib(), "group", dims, mode)


def test_cta_program_runtime_shape():
    _check(_lib(), "block", (7, 3, 2, 2, 6), 1)


def test_leg_mode():
    _check(_lib(), "legs", (4, 2, 2, 2, 8), 1, legs=3, gains=False)


def test_dense_program():
    _check(_lib(), "dense", (5, 3, 2, 2, 6), 1, gains=False)
