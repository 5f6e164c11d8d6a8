"""Parametric handles (nth > 0) and the parallel solver's legs on the device against the extended-precision
restatement (tests/hp_reference.py: solve_parametric, solve_legs) at the conditioning-aware bar of
tests/test_gpu_hp_reference.py: e_kernel <= max(16 e_oracle, 64 u) for every family, the theta families and
collapse_feedback's gain included.

The CTA-per-instance kernel is persistent: its CTAs stride over the instances (or, in leg mode, the legs).  Every
batch here is past that grid, each instance its own problem and theta, and the instances checked sit on both sides of
the first and second strides, so an instance that sees anything of the one its CTA swept before fails."""
import functools

import numpy as np
import pytest

import hp_reference as hp
import lq_cases
import lq_gpu
from lq_cases import PARAM_CASES

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    return lq_gpu.gpu_env()


def outputs(gar, keys):
    return {k: getattr(gar, "OUT_" + k.upper()) for k in keys}


PARAM_OUT = ("ff", "fb", "Vxx", "vx", "ffT", "fbT", "kkt0", "xs", "us", "vs", "vsT", "lbd0", "lbdas", "fth", "Vxt",
             "Vtt", "vt", "kkt0fth", "thGrad", "thHess")
TRAJ_OUT = ("xs", "us", "vs", "vsT", "lbd0", "lbdas")


def grid_of(gar, nx, nu, nc, nct, nc0, N, **kw):
    """The persistent grid of the CTA-per-instance kernel for these dimensions (a batch far past it)."""
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, 1 << 14, **kw)
    g = s.kernel_info()["grid"]
    s.close()
    assert 0 < g < 1 << 14
    return g


def sample(grid, B):
    return sorted({0, grid - 1, grid, grid + 1, 2 * grid, B - 1})


@functools.lru_cache(maxsize=None)
def param_batch(name):
    """(problems, thetas, sampled instances, restatement on them, oracle's error families on them) for a batch of
    2 grid + 3 instances of case `name`."""
    import aligator_b200.gar as gar
    (nx, nu, nc, nct, nth, N), _, mueq, _, nc0, _ = PARAM_CASES[name]
    probs, thetas = lq_cases.param_problems(name, B=1)
    grid = grid_of(gar, nx, nu, nc, nct, probs[0].nc0, N, nth=nth)
    B = 2 * grid + 3
    probs, thetas = lq_cases.param_problems(name, B=B)
    idx = sample(grid, B)
    sub = [probs[b] for b in idx]
    ref, _ = hp.solve_parametric_batch(sub, mueq, thetas[idx])
    return probs, thetas, idx, ref, lq_cases.param_oracle_errors(sub, mueq, thetas[idx], ref)


def run_parametric(gar, name, probs, mueq, thetas, per_instance):
    """backward (or backward_v) + forward_theta on a parametric handle -> every output, and the handle."""
    nx, nu, nc, nct, nth, N = PARAM_CASES[name][0]
    B = len(probs)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, probs[0].nc0, N, B, nth=nth)
    s.set_problem(*gar.pack_problems(probs))
    s.backward(np.full(B, mueq) if per_instance else mueq)
    s.forward(theta=thetas)
    assert np.all(s.status() == 0), s.status()
    return {k: s.get(w).copy() for k, w in outputs(gar, PARAM_OUT).items()}, s


@pytest.mark.parametrize("per_instance", [False, True], ids=["backward", "backward_v"])
@pytest.mark.parametrize("name", list(PARAM_CASES))
def test_parametric_handle_against_extended_precision(env, name, per_instance):
    gar, _, _ = env
    (nx, nu, nc, nct, nth, N), _, mueq, _, _, _ = PARAM_CASES[name]
    probs, thetas, idx, ref, e_oracle = param_batch(name)
    got, s = run_parametric(gar, name, probs, mueq, thetas, per_instance)
    s.close()
    got = {k: v[idx] for k, v in got.items()}
    e_kernel = hp.error_families(got, ref, nu, nc, N)
    assert {"Vxt", "Vtt", "vt", "kkt0fth", "thGrad", "thHess"} <= set(e_kernel)
    title = "parametric %s %s, batch %d, instances %s" % (name, "backward_v" if per_instance else "backward",
                                                          len(probs), idx)
    print("\n" + hp.table(title, e_oracle, e_kernel))
    lq_cases.check_bar(e_kernel, e_oracle, title)


@pytest.mark.parametrize("name", ["c3_gv", "nth33", "G0_nc0_3"])
def test_theta_from_device_memory_and_plain_forward_after_theta(env, name):
    """forward_theta with theta in device memory returns the rollout of theta in host memory bit for bit, and a plain
    forward() after forward_theta(theta) returns the theta-free rollout bit for bit."""
    import ctypes as C
    gar, _, torch = env
    (nx, nu, nc, nct, nth, N), _, mueq, _, _, _ = PARAM_CASES[name]
    probs, thetas, idx, _, _ = param_batch(name)
    host, s = run_parametric(gar, name, probs, mueq, thetas, False)
    traj = outputs(gar, TRAJ_OUT)
    th = torch.from_numpy(np.ascontiguousarray(thetas)).cuda()
    gar._check(gar.lib().ab2_gar_forward_theta(s.h, C.c_void_p(th.data_ptr()), gar.AB2_DEVICE, C.c_void_p(0)))
    s.synchronize()
    for k, w in traj.items():
        assert np.array_equal(s.get(w), host[k]), k
    s.forward()
    free = {k: s.get(w).copy() for k, w in traj.items()}
    s.close()
    fresh = gar.CudaRiccatiBatch(nx, nu, nc, nct, probs[0].nc0, N, len(probs), nth=nth)
    fresh.set_problem(*gar.pack_problems(probs))
    fresh.backward(mueq)
    fresh.forward()
    for k, w in traj.items():
        assert np.array_equal(free[k], fresh.get(w)), k
    fresh.close()
    if nth and np.any(thetas):
        assert not np.array_equal(free["xs"], host["xs"])


# (nx, nu, nc, nct, nc0, N, legs, mueq): C4 dims x 8 legs, C2 dims x 6 legs, nc > 0 with nct > 0
LEG_CASES = [(14, 7, 0, 0, 14, 40, 8, 1e-9), (12, 6, 0, 0, 12, 30, 6, 1e-9), (4, 2, 2, 2, 2, 13, 3, 1e-3)]


@pytest.mark.parametrize("shape", LEG_CASES, ids=["nx%d_nu%d_nc%d_nct%d_nc0%d_N%d_legs%d" % c[:7] for c in LEG_CASES])
def test_leg_handle_against_extended_precision(env, shape):
    """Every factor family of every knot of every leg and collapse_feedback's first gain, with batch * legs past the
    grid: the instances whose legs straddle the first and second strides, against the leg restatement."""
    import gen
    gar, _, _ = env
    nx, nu, nc, nct, nc0, N, T, mueq = shape
    grid = grid_of(gar, nx, nu, nc, nct, nc0, N, legs=T)
    B = (2 * grid + 3 + T - 1) // T
    probs = gen.generate_batch(500 + N + T, B, N, nx, nu, nc, nct)
    if nc0 != nx:
        gen.general_initial_condition(probs, nc0, 15)
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, legs=T)
    s.set_problem(*gar.pack_problems(probs))
    s.backward(mueq)
    s.forward()
    assert np.all(s.status() == 0), s.status()
    keys = ("ff", "fb", "Vxx", "vx", "ffT", "fbT", "fth", "Vxt", "Vtt", "vt") + TRAJ_OUT
    got = {k: s.get(w).copy() for k, w in outputs(gar, keys).items()}
    s.collapse_feedback()
    got["collapse"] = s.get(gar.OUT_FB)[:, 0, :nu].copy()
    s.close()
    idx = sorted({0, (grid - 1) // T, grid // T, (grid + 1) // T, (2 * grid) // T, B - 1})
    sub = [probs[b] for b in idx]
    ref, _ = hp.solve_legs_batch(sub, mueq, T)
    e_oracle = hp.error_families(lq_cases.oracle_legs(sub, mueq, T), ref, nu, nc, N, lq_cases.LEG_FAMILIES)
    e_kernel = hp.error_families({k: v[idx] for k, v in got.items()}, ref, nu, nc, N, lq_cases.LEG_FAMILIES)
    assert {"Kth", "Vxt", "Vtt", "vt", "collapse"} <= set(e_kernel)
    title = "legs %s, batch %d x %d legs (grid %d), instances %s" % (shape, B, T, grid, idx)
    print("\n" + hp.table(title, e_oracle, e_kernel))
    lq_cases.check_bar(e_kernel, e_oracle, title)
