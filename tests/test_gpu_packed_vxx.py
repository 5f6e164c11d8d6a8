"""Vxx of the warp-per-instance sweep is stored as packed lower triangles plus a full slot-0 array
(aligator_b200/csrc/vxx_layout.h, documented at ab2_gar_device_ptr in gar.h).  Every way out of the
handle must still give the full column-major blocks the oracle computes."""
import numpy as np
import pytest

import gen
from oracle import gar_oracle as orc
from oracle import fddp as of

pytestmark = pytest.mark.gpu

TOL = 1e-10


@pytest.fixture(scope="module")
def gar():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import __graft_entry__ as g
    g.build()
    import aligator_b200.gar as gar
    return gar


def _problem(gar, nx, nu, N, B, seed):
    probs = gen.generate_batch(seed, B, N, nx, nu, 0, 0)
    packed = gar.pack_problems(probs)
    bo = orc.BatchedOracle(nx, nu, 0, 0, nx, N, B, *packed)
    bo.sweep(1e-8)
    return probs, packed, bo.get()


class _DeviceArray:
    """A raw device pointer of n doubles, readable by torch.as_tensor."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = dict(shape=(n,), typestr="<f8", data=(ptr, False), version=2)


def _expand(raw, B, N, nx):
    """The documented raw layout: [B][N+1][P] packed lower triangles (column by column), then [B][nx*nx]."""
    P = (nx * (nx + 1) // 2 + 1) & ~1
    pk = raw[:B * (N + 1) * P].reshape(B, N + 1, P)
    V = np.empty((B, N + 1, nx, nx))
    for t in range(N + 1):
        for j in range(nx):
            for i in range(nx):
                a, b = max(i, j), min(i, j)
                V[:, t, i, j] = pk[:, t, b * nx - b * (b - 1) // 2 + (a - b)]
    V[:, 0] = raw[B * (N + 1) * P:B * (N + 1) * P + B * nx * nx].reshape(B, nx, nx).transpose(0, 2, 1)
    return V


@pytest.mark.parametrize("shape", [(12, 6, 40, 9), (14, 7, 20, 5), (6, 3, 30, 7), (4, 2, 0, 3)])
def test_getters_and_raw_layout(gar, shape):
    import torch
    nx, nu, N, B = shape
    probs, packed, ref = _problem(gar, nx, nu, N, B, 40 + nx)
    s = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B)
    s.set_problem(*packed)
    s.sweep(1e-8)
    V = s.get(gar.OUT_VXX)
    assert gen.rel_fro(V, ref["Vxx"]) <= TOL
    dev = torch.empty(B * (N + 1) * nx * nx, dtype=torch.float64, device="cuda:0")
    s.get_into(gar.OUT_VXX, dev.data_ptr(), gar.AB2_DEVICE)
    s.synchronize()
    assert np.array_equal(dev.cpu().numpy().reshape(B, N + 1, nx, nx).transpose(0, 1, 3, 2), V)
    b0, nb, t0, nt = 1, B - 2, N // 2, N + 1 - N // 2
    host = np.empty(nb * nt * nx * nx)
    s.get_range_into(gar.OUT_VXX, b0, nb, t0, nt, host, gar.AB2_HOST)
    dr = torch.empty(nb * nt * nx * nx, dtype=torch.float64, device="cuda:0")
    s.get_range_into(gar.OUT_VXX, b0, nb, t0, nt, dr.data_ptr(), gar.AB2_DEVICE)
    s.synchronize()
    for a in (host, dr.cpu().numpy()):
        assert np.array_equal(a.reshape(nb, nt, nx, nx).transpose(0, 1, 3, 2), V[b0:b0 + nb, t0:t0 + nt])
    P = (nx * (nx + 1) // 2 + 1) & ~1
    n = B * (N + 1) * P + B * nx * nx
    raw = torch.as_tensor(_DeviceArray(s.device_ptr(gar.OUT_VXX), n), device="cuda:0")
    torch.cuda.synchronize()
    assert np.array_equal(_expand(raw.cpu().numpy(), B, N, nx), V)  # the documented raw layout, by hand
    s.close()


def test_get_range_after_cycle_append(gar):
    import torch
    nx, nu, N, B = 12, 6, 9, 4
    probs, packed, ref = _problem(gar, nx, nu, N, B, 5)
    s = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B)
    s.set_problem(*packed)
    s.sweep(1e-8)
    V0 = s.get(gar.OUT_VXX).copy()
    rng = np.random.default_rng(2)
    for cyc in range(1, 3):
        new = [gen.generate_knot(rng, nx, nu, 0, conditioned=True) for _ in range(B)]
        s.cycle_append(np.stack([gar.pack_stage_knot(k, s.srec) for k in new]))
        V = s.get(gar.OUT_VXX)
        assert np.array_equal(V[:, :N - cyc], V0[:, cyc:N]) and np.all(V[:, N - cyc:N] == 0)
        assert np.array_equal(V[:, N], V0[:, N])
        t0, nt = N - cyc - 3, 5  # straddles the wrap point and the zeroed slots
        host = np.empty(2 * nt * nx * nx)
        s.get_range_into(gar.OUT_VXX, 1, 2, t0, nt, host, gar.AB2_HOST)
        dr = torch.empty(2 * nt * nx * nx, dtype=torch.float64, device="cuda:0")
        s.get_range_into(gar.OUT_VXX, 1, 2, t0, nt, dr.data_ptr(), gar.AB2_DEVICE)
        s.synchronize()
        for a in (host, dr.cpu().numpy()):
            assert np.array_equal(a.reshape(2, nt, nx, nx).transpose(0, 1, 3, 2), V[1:3, t0:t0 + nt])
    s.close()


@pytest.mark.parametrize("nchunks", [1, 3])
def test_sweep_host_downloads_vxx(gar, nchunks):
    nx, nu, N, B = 12, 6, 25, 7
    probs, packed, ref = _problem(gar, nx, nu, N, B, 8)
    s = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B)
    V = np.full(B * (N + 1) * nx * nx, np.nan)
    X = np.full(B * (N + 1) * nx, np.nan)
    s.sweep_host(*packed, 1e-8, {gar.OUT_VXX: V, gar.OUT_XS: X}, nchunks=nchunks)
    s.synchronize()
    assert gen.rel_fro(V.reshape(B, N + 1, nx, nx).transpose(0, 1, 3, 2), ref["Vxx"]) <= TOL
    assert gen.rel_fro(X.reshape(B, N + 1, nx), ref["xs"]) <= TOL
    assert np.array_equal(V.reshape(B, N + 1, nx, nx).transpose(0, 1, 3, 2), s.get(gar.OUT_VXX))
    s.close()


@pytest.mark.parametrize("first,second", [(7, 9), (9, 7), (-1, 9)])
def test_variant_switch_between_backward_and_forward(gar, first, second):
    """The forward reads Vxx in the layout the backward wrote, whatever the tuning is by then."""
    nx, nu, N, B = 12, 6, 30, 6
    probs, packed, ref = _problem(gar, nx, nu, N, B, 9)
    s = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B, variant=first)
    s.set_problem(*packed)
    s.backward(1e-8)
    gar.lib().ab2_gar_set_tuning(s.h, gar.C.byref(gar.GarTuning(second, 0, 0)))
    s.forward()
    for key, what in (("Vxx", gar.OUT_VXX), ("xs", gar.OUT_XS), ("us", gar.OUT_US), ("lbdas", gar.OUT_LBDAS)):
        assert gen.rel_fro(s.get(what), ref[key]) <= TOL, key
    s.close()


def test_fddp_vx_reads_either_layout(gar):
    import torch
    from test_fddp import _random_fddp
    nx, nu, N, B = 12, 6, 15, 4
    d = _random_fddp(np.random.default_rng(3), B, N, nx, nu)
    dev = torch.device("cuda:0")
    cm = lambda a: np.ascontiguousarray(np.swapaxes(a, -1, -2))
    arr = {k: torch.tensor(cm(d[k]) if d[k].ndim >= 3 and k not in ("fs", "Lx", "Lu", "Lx_N") else d[k], device=dev)
           for k in d}
    for variant in (-1, 9):
        s = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B, variant=variant)
        Vx = torch.empty(B, N + 1, nx, dtype=torch.float64, device=dev)
        s.fddp_backward_pass(arr, 1e-4, Vx, None)
        s.synchronize()
        Vx = Vx.cpu().numpy()
        for b in range(B):
            r = of.backward_pass(list(d["Jx"][b]), list(d["Ju"][b]), list(d["fs"][b]), list(d["Lxx"][b]),
                                 list(d["Lxu"][b]), list(d["Luu"][b]), list(d["Lx"][b]), list(d["Lu"][b]),
                                 d["Lxx_N"][b], d["Lx_N"][b], 1e-4)
            for i in range(N + 1):
                assert gen.rel_fro(Vx[b, i], r["Vx"][i]) <= TOL, (variant, b, i)
        s.close()
