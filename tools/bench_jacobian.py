"""Time ab2_gar_adjoint_many and ab2_gar_tangent_many per cotangent / tangent against one ab2_gar_adjoint and one
ab2_gar_tangent call, at C2 (nx12 nu6 N100 B4096, nrhs 1, 4, 8) and C3 (nx4 nu2 nc2 N100 B16384, mu 1e-3, nrhs 1, 8, 32).

    python tools/bench_jacobian.py [--iters 10] [--warmup 3] [--configs C2,C3]

Per config: the single adjoint and tangent calls, then for every nrhs the reverse-mode call and, after its buffers are
freed, the forward-mode call (at C3 and nrhs 32 the gradient records alone take about 33 GB).  Times are ms per call
from CUDA events over `iters` back-to-back calls after `warmup` calls, and ms per right-hand side.  From nrhs 8 up,
a separate torch.profiler run gives each kernel of the two calls its time, and for the two new streaming kernels the
HBM bandwidth their byte count implies (per right-hand side and knot: the record written or read and the rhs vectors;
per knot: the primal vectors).  Prints one JSON line per (config, nrhs), with the card's name and power limit read in
the same run."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_adjoint import CONFIGS, card  # noqa: E402

NRHS = dict(C2=(1, 4, 8), C3=(1, 8, 32))
KEYS = ("xs", "us", "vs", "vsT", "lam0", "lams")


def kernel_bytes(nx, nu, nc, srec, B, N, nrhs):
    """HBM bytes each new streaming kernel moves (stage knots; terminal knots, G0 and g0 are < 1 % at N = 100)."""
    vec = 2 * nx + nu + nc  # x_t, u_t, v_t, lambda_{t+1}: the primal once per knot, y or rho once per rhs and knot
    per = 8 * B * N * (nrhs * (srec + vec) + vec)
    return dict(grad=per, rhs=per)


def timed(torch, f, iters, warmup):
    for _ in range(warmup):
        f()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def profiled(torch, f):
    """ms per call of each kernel of f, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            f()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        if ev.device_type.name != "CUDA" or ev.count == 0:
            continue
        t = getattr(ev, "device_time_total", None) or ev.cuda_time_total
        key = ("grad" if "jacobian_grad" in ev.key else "rhs" if "jacobian_rhs" in ev.key
               else "resolve" if "resolve_kernel" in ev.key else None)
        if key:
            kern[key] = kern.get(key, 0.0) + t / 3 / 1e3
    return kern


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--configs", default="C2,C3")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    import aligator_b200.gar as gar
    import bench
    name, power = card()
    for cfg, nx, nu, nc, nct, N, B, mu in CONFIGS:
        if cfg not in args.configs.split(","):
            continue
        stage, term, G0, g0 = bench.synth_batch_torch(torch, B, N, nx, nu, "cuda:0", 7, nc, nct, "control")
        s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nx, N, B)
        s.set_problem(stage, term, G0, g0, memspace=gar.AB2_DEVICE)
        s.sweep(mu)
        outs = dict(xs=gar.OUT_XS, us=gar.OUT_US, vs=gar.OUT_VS, vsT=gar.OUT_VST, lam0=gar.OUT_LBD0, lams=gar.OUT_LBDAS)
        primal = {}
        for k, w in outs.items():
            primal[k] = torch.empty(s.out_shape(w), dtype=torch.float64, device="cuda")
            if primal[k].numel():
                s.get_into(w, primal[k], gar.AB2_DEVICE)
        rec = dict(stage=stage, term=term, G0=G0, g0=g0)
        # one cotangent / tangent per call, in the same run
        cot1 = {k: torch.randn_like(v) for k, v in primal.items()}
        grad1 = {k: torch.empty_like(v) for k, v in rec.items()}
        dot1 = {k: torch.randn_like(v) for k, v in rec.items()}
        adj_ms = timed(torch, lambda: s.adjoint(primal, cot1, grad1, mu), args.iters, args.warmup)
        tan_ms = timed(torch, lambda: s.tangent(primal, dot1, mu), args.iters, args.warmup)
        del cot1, grad1, dot1
        s.sweep(mu)  # the factorisation the calls below re-solve on (the adjoint and tangent calls leave the same one)
        for nrhs in NRHS[cfg]:
            row = dict(config=cfg, batch=B, horizon=N, nrhs=nrhs, gpu=name, power_limit=power,
                       adjoint_ms=round(adj_ms, 4), tangent_ms=round(tan_ms, 4))
            many = lambda: {k: torch.empty((nrhs,) + tuple(v.shape), dtype=torch.float64, device="cuda")
                            for k, v in primal.items()}
            # reverse mode
            cot = {k: torch.randn((nrhs,) + tuple(v.shape), dtype=torch.float64, device="cuda")
                   for k, v in primal.items()}
            work = many()
            grad = {k: torch.empty((nrhs,) + tuple(v.shape), dtype=torch.float64, device="cuda") for k, v in rec.items()}
            f = lambda: s.adjoint_many(primal, cot, work, grad, mu)
            ms = timed(torch, f, args.iters, args.warmup)
            row.update(adjoint_many_ms=round(ms, 4), adjoint_many_ms_per_rhs=round(ms / nrhs, 4),
                       adjoint_speedup=round(adj_ms / (ms / nrhs), 2))
            kr = profiled(torch, f) if nrhs >= 8 else {}
            del cot, work, grad, f
            s._keep.pop("adjoint_many", None)  # the handle keeps the last call's arrays alive: release them before allocating
            torch.cuda.empty_cache()
            # forward mode
            dot = {k: torch.randn((nrhs,) + tuple(v.shape), dtype=torch.float64, device="cuda") for k, v in rec.items()}
            work, out = many(), many()
            f = lambda: s.tangent_many(primal, dot, work, out, mu)
            ms = timed(torch, f, args.iters, args.warmup)
            row.update(tangent_many_ms=round(ms, 4), tangent_many_ms_per_rhs=round(ms / nrhs, 4),
                       tangent_speedup=round(tan_ms / (ms / nrhs), 2))
            kf = profiled(torch, f) if nrhs >= 8 else {}
            del dot, work, out, f
            s._keep.pop("tangent_many", None)
            torch.cuda.empty_cache()
            if kr or kf:
                by = kernel_bytes(nx, nu, nc, s.srec, B, N, nrhs)
                kt = dict(grad=kr.get("grad"), rhs=kf.get("rhs"))
                row.update(kernel_ms=dict(adjoint_many={k: round(v, 4) for k, v in kr.items()},
                                          tangent_many={k: round(v, 4) for k, v in kf.items()}),
                           kernel_GBps={k: round(by[k] / (t * 1e-3) / 1e9, 1) for k, t in kt.items() if t},
                           kernel_frac_of_3350={k: round(by[k] / (t * 1e-3) / 1e9 / 3350.0, 3)
                                                for k, t in kt.items() if t})
            print(json.dumps(row), flush=True)
        s.close()
        del stage, term, G0, g0, rec, primal
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
