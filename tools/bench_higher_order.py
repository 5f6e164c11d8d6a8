"""Time the higher derivatives of the LQ solve (lq_solve_higher) against one sweep, at C2 (nx12 nu6 N100 B4096) and C3
(nx4 nu2 nc2 N100 B16384, mu 1e-3), for V in {1, 8, 32} directions.

    python tools/bench_higher_order.py [--iters 5] [--warmup 2] [--configs C2,C3] [--dirs 1,8,32]

Per config: one sweep (the yardstick), then per V one Hessian-vector-product batch of a quadratic loss of the solution
with respect to the stage records (torch.func.vmap over V of torch.func.jvp of torch.func.grad: per call two rho
launches, two resolves and one two-pair gradient launch), and torch.func.hessian of the loss with respect to g0 on a
sub-batch of 8 instances (8 nc0 directions).  Times are ms per call from CUDA events over `iters` calls after `warmup`
calls; the HVP includes lq_solve_higher's own sweep.  A separate torch.profiler run of one HVP batch gives each kernel
instantiation its time, and for the streaming kernels the HBM bandwidth their byte count implies (records, and the
per-direction and shared vectors, as each call staged them).  A V that does not fit the card's memory prints
{"oom": true}.  Prints one JSON line per (config, V), with the card's name and power limit read in the same run."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_adjoint import CONFIGS, card  # noqa: E402
from bench_jacobian import timed  # noqa: E402

PEAK_GBPS = 3350.0  # H100 SXM HBM3


def _count_calls(s, log):
    """Record the kernel instantiation and the HBM bytes of every rho_many / grad_many call of s."""
    d = s.dims
    knot = 2 * d.nx + d.nu + d.nc  # x_t, u_t, v_t, lambda_{t+1}
    per_rhs_knot = lambda n: 8 * d.batch * d.horizon * n
    shared = lambda v: v["xs"].numel() == d.batch * (d.horizon + 1) * d.nx
    rho, grad = s.rho_many, s.grad_many

    def rho_many(dot, a, out, vectors=True, dot2=None, a2=None, e=None, stream=0):
        nrhs = out["xs"].numel() // (d.batch * (d.horizon + 1) * d.nx)
        plain = vectors and shared(a) and dot2 is None and e is None
        name = "rhs<%s>" % ("plain" if plain else "ext")
        recs = 1 + (dot2 is not None)
        vecs = 1 + (not shared(a)) + (e is not None) + (dot2 is not None and not shared(a2))
        by = nrhs * per_rhs_knot(recs * s.srec + vecs * knot) + per_rhs_knot(knot) * (shared(a) + (dot2 is not None
                                                                                                    and shared(a2)))
        log.append((name, by))
        return rho(dot, a, out, vectors, dot2, a2, e, stream)

    def grad_many(y, z, g, vectors=True, y2=None, z2=None, stream=0):
        nrhs = y["xs"].numel() // (d.batch * (d.horizon + 1) * d.nx)
        plain = vectors and shared(z) and y2 is None
        name = "grad<%s>" % ("plain" if plain else "ext")
        vecs = 1 + (not shared(z)) + (0 if y2 is None else 1 + (not shared(z2)))
        by = nrhs * per_rhs_knot(s.srec + vecs * knot) + per_rhs_knot(knot) * (shared(z) + (y2 is not None
                                                                                             and shared(z2)))
        log.append((name, by))
        return grad(y, z, g, vectors, y2, z2, stream)
    s.rho_many, s.grad_many = rho_many, grad_many


def _kernel_ms(torch, f):
    """ms of each kernel instantiation in one call of f, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        if ev.device_type.name != "CUDA" or ev.count == 0:
            continue
        t = (getattr(ev, "device_time_total", None) or ev.cuda_time_total) / 1e3
        k = ev.key
        key = ("rhs<ext>" if "jacobian_rhs_kernel<false, true>" in k else
               "rhs<plain>" if "jacobian_rhs_kernel" in k else
               "grad<ext>" if "jacobian_grad_kernel<false, true>" in k else
               "grad<plain>" if "jacobian_grad_kernel" in k else
               "resolve" if "resolve" in k else
               "sweep" if ("riccati" in k or "sweep" in k or "block" in k) else "other")
        kern[key] = kern.get(key, 0.0) + t
    return kern


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--configs", default="C2,C3")
    ap.add_argument("--dirs", default="1,8,32")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    import aligator_b200.autograd as ag
    import aligator_b200.gar as gar
    import bench
    name, power = card()
    F = torch.func
    for cfg, nx, nu, nc, nct, N, B, mu in CONFIGS:
        if cfg not in args.configs.split(","):
            continue
        stage, term, G0, g0 = bench.synth_batch_torch(torch, B, N, nx, nu, "cuda:0", 7, nc, nct, "control")
        s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nx, N, B)
        s.set_problem(stage, term, G0, g0, memspace=gar.AB2_DEVICE)
        sweep_ms = timed(torch, lambda: s.sweep(mu), args.iters, args.warmup)
        gen = torch.Generator(device="cuda").manual_seed(3)
        W = [torch.randn(o.shape, generator=gen, dtype=torch.float64, device="cuda")
             for o in ag.lq_solve(s, stage, term, G0, g0, mu)]
        loss = lambda outs: sum((w * o).sum() + 0.5 * (w * o * o).sum() for w, o in zip(W, outs))
        f = lambda st: loss(ag.lq_solve_higher(s, st, term, G0, g0, mu))
        # torch.func.hessian with respect to g0 on a sub-batch of 8 instances
        sub = [t[:8].contiguous() for t in (stage, term, G0, g0)]
        h8 = gar.CudaRiccatiBatch(nx, nu, nc, nct, nx, N, 8)
        W8 = [w[:8] for w in W]
        f8 = lambda x: sum((w * o).sum() + 0.5 * (w * o * o).sum()
                           for w, o in zip(W8, ag.lq_solve_higher(h8, sub[0], sub[1], sub[2], x, mu)))
        hess_ms = timed(torch, lambda: F.hessian(f8)(sub[3]), args.iters, args.warmup)
        h8.close()
        for V in [int(v) for v in args.dirs.split(",")]:
            row = dict(config=cfg, batch=B, horizon=N, mu=mu, directions=V, gpu=name, power_limit=power,
                       sweep_ms=round(sweep_ms, 4), hessian_g0_sub8_ms=round(hess_ms, 4))
            try:
                dirs = torch.randn((V,) + tuple(stage.shape), generator=gen, dtype=torch.float64, device="cuda")
                hvp = lambda: F.vmap(lambda v: F.jvp(F.grad(f), (stage,), (v,))[1])(dirs)
                ms = timed(torch, hvp, args.iters, args.warmup)
                row.update(hvp_ms=round(ms, 4), hvp_ms_per_direction=round(ms / V, 4),
                           hvp_over_sweep=round(ms / sweep_ms, 2))
                log = []
                _count_calls(s, log)
                kern = _kernel_ms(torch, hvp)
                del s.rho_many, s.grad_many  # back to the class's methods
                by = {}
                for k, b in log:
                    by[k] = by.get(k, 0) + b
                row.update(kernel_ms={k: round(v, 4) for k, v in kern.items()},
                           kernel_GBps={k: round(by[k] / (kern[k] * 1e-3) / 1e9, 1) for k in by if kern.get(k)},
                           kernel_frac_of_3350={k: round(by[k] / (kern[k] * 1e-3) / 1e9 / PEAK_GBPS, 3)
                                                for k in by if kern.get(k)})
                del dirs, hvp
            except torch.cuda.OutOfMemoryError:
                row.update(oom=True)
            s._keep.clear()
            torch.cuda.empty_cache()
            print(json.dumps(row), flush=True)
        s.close()
        del stage, term, G0, g0, W
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
