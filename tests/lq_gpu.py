"""The GPU side of the derivative tests: the module fixture's body, the handle matrix, handle setup, and the buffer
and copy helpers that several GPU test modules share.  torch and aligator_b200 are imported by the fixture."""
import numpy as np

import gen
import lq_cases
import lq_factor_adjoint_ref


def gpu_env():
    """(gar, autograd, torch) after building the package: the body of every GPU module's `env` fixture."""
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import __graft_entry__ as g
    g.build()
    import aligator_b200.gar as gar
    import aligator_b200.autograd as ag
    return gar, ag, torch


MUS = (1.0, 1e-2, 1e-5)
# (name, CudaRiccatiBatch keyword arguments, (nx, nu, nc, nct, nc0, N, B))
HANDLES = [("lane_v%d" % v, dict(variant=v), (4, 2, 2, 2, 4, 6, 9)) for v in range(7)] + [
    ("lane_12_6_6", {}, (12, 6, 6, 3, 12, 5, 7))] + [
    ("mma_12_v%d" % v, dict(variant=v), (12, 6, 0, 3, 12, 6, 9)) for v in (6, 7, 8, 10)] + [
    ("mma_14_v%d" % v, dict(variant=v), (14, 7, 0, 2, 14, 4, 5)) for v in (6, 7, 8, 10)] + [
    ("cta_v9", dict(variant=9), (4, 2, 2, 2, 4, 6, 9)),
    ("cta_runtime", {}, (7, 3, 2, 2, 7, 5, 8)),
    ("dense", dict(dense=True), (4, 2, 2, 2, 4, 5, 8)),
]
SERIAL = [h for h in HANDLES if not h[1].get("dense")]


def setup(env, kw, dims, seed, mu=1e-2):
    """A handle of B seeded problems, swept at mu: (handle, packed records)."""
    gar, _, _ = env
    nx, nu, nc, nct, nc0, N, B = dims
    probs = gen.generate_batch(seed, B, N, nx, nu, nc, nct)
    recs = [np.ascontiguousarray(a) for a in gar.pack_problems(probs)]
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, **kw)
    s.set_problem(*recs)
    s.sweep(mu)
    return s, recs


def _empty(torch, s, w):
    return torch.empty(s.out_shape(w), dtype=torch.float64, device="cuda")


def out_of(gar):
    return dict(xs=gar.OUT_XS, us=gar.OUT_US, vs=gar.OUT_VS, vsT=gar.OUT_VST, lam0=gar.OUT_LBD0, lams=gar.OUT_LBDAS)


def primal(env, s):
    """The handle's trajectory copied into tensors of the caller (what the last sweep returned)."""
    gar, _, torch = env
    out = {}
    for k, w in out_of(gar).items():
        t = _empty(torch, s, w)
        if t.numel():
            s.get_into(w, t, gar.AB2_DEVICE)
        out[k] = t
    s.synchronize()
    return out


def cotangent(env, s, seed, scale=1.0):
    gar, _, torch = env
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return {k: scale * torch.randn(s.out_shape(w), generator=g, dtype=torch.float64, device="cuda")
            for k, w in out_of(gar).items()}


def grad_bufs(env, s, fill=float("nan")):
    _, _, torch = env
    d = s.dims
    shapes = dict(stage=(d.batch, d.horizon, s.srec), term=(d.batch, s.trec), G0=(d.batch, d.nc0 * d.nx),
                  g0=(d.batch, d.nc0))
    return {k: torch.full(v, fill, dtype=torch.float64, device="cuda") for k, v in shapes.items()}


def to_np(d):
    return {k: v.cpu().numpy() for k, v in d.items()}


OUTS_PLAIN = range(13)  # OUT_FF .. OUT_LBDAS


def outputs(gar, s):
    r = {w: s.get(w).copy() for w in OUTS_PLAIN if int(np.prod(s.out_shape(w)))}
    r["status"] = s.status().copy()
    r["pivots"] = np.stack(s.pivot_stats(), axis=1)
    return r


def zeros_like_outputs(env, s):
    gar, _, torch = env
    return {k: torch.zeros(s.out_shape(w), dtype=torch.float64, device="cuda") for k, w in out_of(gar).items()}


def block_inputs(torch, probs):
    """Leaf tensors of every block of a batch, Q and R as P with Q = (P + P^T) / 2."""
    N = probs[0].horizon
    T = lambda f: torch.tensor(np.stack([np.stack([np.asarray(f(p, t)) for t in range(N)]) for p in probs]),
                               dtype=torch.float64, device="cuda", requires_grad=True)
    blocks = {n: T(lambda p, t, n=n: getattr(p.stages[t], n)) for n in ("A", "B", "f", "Q", "S", "R", "q", "r", "C",
                                                                      "D", "d")}
    Tt = lambda f: torch.tensor(np.stack([np.asarray(f(p)) for p in probs]), dtype=torch.float64, device="cuda",
                                requires_grad=True)
    term = {n: Tt(lambda p, n=n: getattr(p.stages[N], n)) for n in ("Q", "q", "C", "d")}
    init = dict(G0=Tt(lambda p: np.asarray(p.G0).ravel(order="F")), g0=Tt(lambda p: p.g0))
    return blocks, term, init


def rec_shapes(s):
    d = s.dims
    return dict(stage=(d.batch, d.horizon, s.srec), term=(d.batch, s.trec), G0=(d.batch, d.nc0 * d.nx),
                g0=(d.batch, d.nc0))


def _randn(torch, shape, seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return torch.randn(shape, generator=g, dtype=torch.float64, device="cuda")


def cots(env, s, primal, nrhs, seed):
    return {k: _randn(env[2], (nrhs,) + tuple(v.shape), seed + i) for i, (k, v) in enumerate(primal.items())}


def dots(env, s, nrhs, seed):
    return {k: _randn(env[2], (nrhs,) + sh, seed + i) for i, (k, sh) in enumerate(rec_shapes(s).items())}


def _nan(torch, shape):
    return torch.full(shape, float("nan"), dtype=torch.float64, device="cuda")


def sol_bufs(env, primal, nrhs):
    return {k: _nan(env[2], (nrhs,) + tuple(v.shape)) for k, v in primal.items()}


def grad_bufs_many(env, s, nrhs):
    return {k: _nan(env[2], (nrhs,) + sh) for k, sh in rec_shapes(s).items()}


def handle_records(gar, probs):
    stage, term, G0, g0 = [np.ascontiguousarray(a) for a in gar.pack_problems(probs)]
    B, N = len(probs), probs[0].horizon
    return stage.reshape(B, N, stage.size // max(B * N, 1)), term.reshape(B, -1), G0.reshape(B, -1), g0.reshape(B, -1)


def factor(gar, s):
    """The handle's own factorisation in the restatement's shapes."""
    return dict(ff=s.get(gar.OUT_FF), fb=s.get(gar.OUT_FB), vxx=s.get(gar.OUT_VXX), vx=s.get(gar.OUT_VX),
                fft=s.get(gar.OUT_FFT), fbt=s.get(gar.OUT_FBT))


def dev(torch, a):
    return None if a is None else torch.tensor(np.ascontiguousarray(a, dtype=np.float64), device="cuda")


def grads(torch, s):
    d = s.dims
    shapes = dict(stage=(d.batch, d.horizon, s.srec), term=(d.batch, s.trec), G0=(d.batch, d.nc0 * d.nx),
                  g0=(d.batch, d.nc0))
    return {k: torch.full(v, float("nan"), dtype=torch.float64, device="cuda") for k, v in shapes.items()}


def device_factor_adjoint(env, s, cot, mu, d6):
    """ab2_gar_factor_adjoint of the handle on the restatement-shaped cotangent `cot`: the gradient records."""
    _, _, torch = env
    dc = {k: dev(torch, v) for k, v in lq_cases.device_cot(cot, d6, s.dims.batch).items()}
    g = grads(torch, s)
    s.factor_adjoint(dc, g, mu if np.ndim(mu) == 0 else dev(torch, mu))
    s.synchronize()
    return {k: v.cpu().numpy() for k, v in g.items()}


def outs(torch, case, B):
    """NaN-filled out tensors in the device layouts (vxx as column-major blocks: same shape)."""
    return {k: torch.full(s, float("nan"), dtype=torch.float64, device="cuda")
            for k, s in lq_cases.out_shapes(case, B).items()}


def device_factor_tangent(env, s, dot, mu, d6, want=lq_factor_adjoint_ref.COT):
    """ab2_gar_factor_tangent of the handle along the record tangent `dot`, only `want` written: the restatement's
    shapes."""
    _, _, torch = env
    B = s.dims.batch
    o = outs(torch, d6, B)
    s.factor_tangent({k: dev(torch, v) for k, v in dot.items()}, {k: v for k, v in o.items() if k in want},
                     mu if np.ndim(mu) == 0 else dev(torch, mu))
    s.synchronize()
    return {k: (np.swapaxes(v.cpu().numpy(), -1, -2) if k == "vxx" else v.cpu().numpy()) for k, v in o.items()}


# (name, CudaRiccatiBatch keyword arguments, (nx, nu, nc, nct, nc0, N, B), mu)
FACTOR_HANDLES = [("warp_c3", {}, (4, 2, 2, 2, 4, 6, 9), 1e-3),
                  ("cta_v9", dict(variant=9), (4, 2, 2, 2, 4, 6, 9), 1e-3),
                  ("mma_12", {}, (12, 6, 0, 3, 12, 6, 9), 1e-3),
                  ("lane_c1", {}, (6, 3, 0, 2, 3, 5, 5), 1e-3),
                  ("cta_runtime", {}, (7, 3, 2, 2, 7, 5, 8), 1e-2),
                  ("N0", {}, (4, 2, 2, 2, 4, 0, 3), 1e-3),
                  ("N1", {}, (6, 3, 0, 2, 3, 1, 3), 1e-3),
                  ("small_mu", {}, (4, 2, 2, 2, 4, 5, 4), 1e-8),
                  ("small_mu_v9", dict(variant=9), (12, 6, 0, 3, 12, 4, 3), 1e-8)]


class DeviceArray:
    """A raw device pointer of n doubles, readable by torch.as_tensor."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = dict(shape=(n,), typestr="<f8", data=(ptr, False), version=2)
