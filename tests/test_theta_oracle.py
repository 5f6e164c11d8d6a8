"""The theta-derivative programs of parametric problems (aligator_b200/csrc/lq_theta.cuh: ab2_gar_theta_tangent, J d,
and ab2_gar_theta_adjoint, J^T zbar), executed on the CPU through the host emulation on the factors of the emulated
parametric sweep.  Checked against the extended-precision Jacobian (lq_theta_ref.theta_jacobian: the reference's
rollout without its feed-forward terms, started at kkt0fth) at the bar e_kernel <= max(16 e_oracle, 64 u), where
e_oracle is the error of the same recursion in fp64 numpy on the oracle's factors (tests/lq_theta_ref.py); and for
exact transposition, consistency with the parametric forward pass, bit-for-bit invariance of a direction's result,
and the shared-memory size of every served shape."""
import ctypes as C
import functools

import numpy as np
import pytest

import hp_reference as hp
import lq_cases
import lq_theta_ref as tref
from emu_harness import emulate
from theta_emu_harness import SOL as THETA_SOL, lib, run_theta, shapes as theta_shapes
from lq_cases import PARAM_CASES

# nth in {1, nx, 33}, terminal Gv and constraints, N 0 and 1, nc0 in {0, 1, nx/2, nx}, mu 1e-3 and 1e-8
CASES = ["c3_mu1e-3", "c3_mu1e-8", "nct_gv", "nth1", "nth_nx", "nth33", "N0", "N1", "theta1e6",
         "G0_nc0_0", "G0_nc0_1", "G0_nc0_3", "G0_nc0_6"]
NRHS = 3


def warps(nx, nu, nc, nth):
    """The fewest emulated warps the parametric sweep program runs these dimensions on."""
    return (max(nx + 1, nu + nc, 2 * nx, nu + nc + nx, nth) + 31) // 32


def d7_of(name):
    (nx, nu, nc, nct, nth, N), B, mueq, _, _, _ = PARAM_CASES[name]
    nc0 = lq_cases.param_problems(name)[0][0].nc0
    return (nx, nu, nc, nct, nc0, nth, N), B, mueq


@functools.lru_cache(maxsize=None)
def case(name):
    """(problems, thetas, raw emulated factors, oracle factors per instance, extended-precision J per instance)."""
    d7, B, mueq = d7_of(name)
    nx, nu, nc, nct, nc0, nth, N = d7
    probs, thetas = lq_cases.param_problems(name)
    raw = emulate("parametric", probs, (nx, nu, nc, nct, N), mueq, warps(nx, nu, nc, nth), nth=nth,
                  theta=np.ascontiguousarray(thetas))
    assert np.all(raw["status"] == 0), raw["status"]
    o = lq_cases.oracle_parametric(probs, mueq, thetas)
    fac = [{k: o[k][b] for k in ("fb", "fth", "Vxx", "Vxt", "kkt0fth", "fbT")} for b in range(B)]
    J = [tref.theta_jacobian(p, mueq) for p in probs]
    return probs, thetas, raw, fac, J


def _rename(z):
    """The kernel's field names -> hp_reference's (lam0 -> lbd0, lams -> lbdas)."""
    m = dict(lam0="lbd0", lams="lbdas")
    return {m.get(k, k): v for k, v in z.items()}


def _flat(z):
    """[nrhs][B][...] fields -> [nrhs*B][...] (directions as instances)."""
    return {k: v.reshape((v.shape[0] * v.shape[1],) + v.shape[2:]) for k, v in z.items()}


def directions(name, seed=1):
    d7, B, _ = d7_of(name)
    return np.random.default_rng(seed).standard_normal((NRHS, B, d7[5]))


def cotangents(name, seed=2):
    d7, B, _ = d7_of(name)
    rng = np.random.default_rng(seed)
    return {k: rng.standard_normal((NRHS,) + s) for k, s in theta_shapes(d7, B).items()}


@pytest.mark.parametrize("name", CASES)
def test_tangent_against_extended_precision(name):
    d7, B, _ = d7_of(name)
    nx, nu, nc, nct, nc0, nth, N = d7
    _, _, raw, fac, J = case(name)
    d = directions(name)
    got = _flat(_rename(run_theta(raw, d7, 32, NRHS, dtheta=d)))
    per = [(j, b) for j in range(NRHS) for b in range(B)]
    ref = hp.stack_solutions([tref.jacobian_apply(J[b], d[j, b]) for j, b in per])
    ora = hp.stack_solutions([tref.tangent(fac[b], d[j, b], nu, nc) for j, b in per])
    e_kernel, e_oracle = tref.errors(got, ref, nu, nc, N), tref.errors(ora, ref, nu, nc, N)
    assert {"xs", "us", "lbd"} <= set(e_kernel) or N == 0
    print("\n" + hp.table("theta_tangent %s" % name, e_oracle, e_kernel))
    lq_cases.check_bar(e_kernel, e_oracle, "theta_tangent %s" % name)


@pytest.mark.parametrize("name", CASES)
def test_adjoint_against_extended_precision(name):
    d7, B, _ = d7_of(name)
    nx, nu, nc, nct, nc0, nth, N = d7
    _, _, raw, fac, J = case(name)
    z = cotangents(name)
    got = run_theta(raw, d7, 32, NRHS, cot=z)["theta_bar"].reshape(-1, nth)
    zr = _rename(z)
    per = [(j, b) for j in range(NRHS) for b in range(B)]
    pick = lambda j, b: {k: v[j, b] for k, v in zr.items()}
    ref = np.stack([tref.jacobian_transpose_apply(J[b], pick(j, b)) for j, b in per])
    ora = np.stack([tref.adjoint(fac[b], pick(j, b), nu, nc) for j, b in per])
    e_kernel, e_oracle = tref.theta_errors(got, ref), tref.theta_errors(ora, ref)
    print("\n" + hp.table("theta_adjoint %s" % name, e_oracle, e_kernel))
    lq_cases.check_bar(e_kernel, e_oracle, "theta_adjoint %s" % name)


@pytest.mark.parametrize("name", CASES)
def test_adjoint_is_the_transpose(name):
    """<zbar, J d> = <J^T zbar, d> to rounding, the two sides from the two emulated programs."""
    d7, B, _ = d7_of(name)
    _, _, raw, _, _ = case(name)
    d, z = directions(name, 3), cotangents(name, 4)
    jd = run_theta(raw, d7, 32, NRHS, dtheta=d)
    tb = run_theta(raw, d7, 32, NRHS, cot=z)["theta_bar"]
    for j in range(NRHS):
        for b in range(B):
            terms = np.concatenate([(z[k][j, b] * jd[k][j, b]).ravel() for k in THETA_SOL])
            lhs, rhs = terms.sum(), float(tb[j, b] @ d[j, b])
            scale = np.abs(terms).sum() + np.abs(tb[j, b] * d[j, b]).sum()
            assert abs(lhs - rhs) <= 1e-12 * scale, (j, b, lhs, rhs, scale)


@pytest.mark.parametrize("name", ["c3_mu1e-3", "nct_gv", "nth33", "N0", "N1", "G0_nc0_3"])
def test_tangent_is_the_difference_of_two_forward_passes(name):
    """The emulated parametric forward at theta + d minus at theta equals J d, within the rounding of the two
    rollouts (a few ulps of their size per family, times the horizon)."""
    d7, B, mueq = d7_of(name)
    nx, nu, nc, nct, nc0, nth, N = d7
    probs, thetas, raw, _, _ = case(name)
    d = directions(name, 5)[0]
    hi = emulate("parametric", probs, (nx, nu, nc, nct, N), mueq, warps(nx, nu, nc, nth), nth=nth,
                 theta=np.ascontiguousarray(thetas + d))
    jd = run_theta(raw, d7, 32, 1, dtheta=d[None])
    outs = dict(xs="xs", us="us", vs="vs", vsT="vsT", lam0="lbd0", lams="lbdas")
    for k, ok in outs.items():
        if not jd[k][0].size:
            continue
        a, b0 = hi[ok].reshape(jd[k][0].shape), raw[ok].reshape(jd[k][0].shape)
        bound = 64 * hp.U * max(N, 1) * (np.abs(a).max() + np.abs(b0).max())
        assert np.abs((a - b0) - jd[k][0]).max() <= bound, (k, np.abs((a - b0) - jd[k][0]).max(), bound)


@pytest.mark.parametrize("name", ["c3_gv", "nth33", "N0"])
def test_direction_is_bit_identical_across_nrhs_chunk_lanes_and_position(name):
    d7, B, _ = d7_of(name)
    _, _, raw, _, _ = case(name)
    rng = np.random.default_rng(9)
    d = rng.standard_normal((5, B, d7[5]))
    z = {k: rng.standard_normal((5,) + s) for k, s in theta_shapes(d7, B).items()}
    base_t = run_theta(raw, d7, 32, 5, dtheta=d)
    base_a = run_theta(raw, d7, 32, 5, cot=z)["theta_bar"]
    perm = [3, 0, 4, 1, 2]
    for lanes, chunk in ((1, 1), (7, 2), (32, 5), (5, 3)):
        t = run_theta(raw, d7, lanes, chunk, dtheta=np.ascontiguousarray(d[perm]))
        a = run_theta(raw, d7, lanes, chunk, cot={k: np.ascontiguousarray(v[perm]) for k, v in z.items()})["theta_bar"]
        for k in THETA_SOL:
            assert np.array_equal(t[k], base_t[k][perm]), (lanes, chunk, k)
        assert np.array_equal(a, base_a[perm]), (lanes, chunk)
    one = run_theta(raw, d7, 32, 1, dtheta=np.ascontiguousarray(d[2:3]))
    for k in THETA_SOL:
        assert np.array_equal(one[k][0], base_t[k][2]), k
    one = run_theta(raw, d7, 32, 1, cot={k: np.ascontiguousarray(v[2:3]) for k, v in z.items()})["theta_bar"]
    assert np.array_equal(one[0], base_a[2])


def test_missing_cotangent_fields_are_zero():
    name = "nct_gv"
    d7, B, _ = d7_of(name)
    _, _, raw, _, _ = case(name)
    z = cotangents(name)
    zero = {k: (np.zeros_like(v) if k in ("us", "vsT", "lam0") else v) for k, v in z.items()}
    part = {k: v for k, v in z.items() if k not in ("us", "vsT", "lam0")}
    assert np.array_equal(run_theta(raw, d7, 32, NRHS, cot=part)["theta_bar"],
                          run_theta(raw, d7, 32, NRHS, cot=zero)["theta_bar"])


def test_every_served_shape_fits_or_is_refused():
    """Every shape the library accepts (ab2_gar_supported; nct in {0, nx}, nth in {1, nx, 33}) with nx, nu, nc < 80:
    one direction's item fits 227 KB of shared memory, or it is among the shapes the calls refuse with
    AB2_ERR_UNSUPPORTED (the same size function).  The dimensions of the parametric cases served in practice fit."""
    import aligator_b200.gar as gar
    e = lib()
    fn = C.CFUNCTYPE(C.c_int, C.c_int, C.c_int, C.c_int, C.c_int)(lambda nx, nu, nc, nc0: gar.supported(nx, nu, nc, nc0))
    bad = (C.c_int * 6)()
    largest, accepted = C.c_long(0), C.c_long(0)
    over = e.emu_theta_size_scan(C.cast(fn, C.c_void_p), 80, bad, C.byref(largest), C.byref(accepted))
    print("\naccepted %d, over 227 KB %d (first %s), largest fitting item %d bytes"
          % (accepted.value, over, list(bad), largest.value))
    assert accepted.value > 0 and 0 < largest.value <= 227 * 1024
    if over:
        nx, nu, nc, nc0, nct, nth = bad
        assert e.emu_theta_item_bytes(nx, nu, nc, nct, nc0, nth, 1) > 227 * 1024
    # C2, C3 and C5 dimensions at the nth the project measures, with terminal constraints
    for nx, nu, nc, nct, nc0, nth in ((12, 6, 0, 0, 12, 12), (4, 2, 2, 2, 4, 2), (57, 28, 0, 0, 57, 4), (12, 6, 0, 12, 12, 33)):
        assert e.emu_theta_item_bytes(nx, nu, nc, nct, nc0, nth, 1) <= 227 * 1024
