"""Time ab2_gar_refine against the handle's own sweep at C2 (nx12 nu6 N100 B4096), C3 (nx4 nu2 nc2 nct2 N100 B16384)
and C5 (nx57 nu28 N150 B512), all at mu 1e-8.

    python tools/bench_refine.py [--iters 20] [--warmup 5]

Per config: ms per refinement step, from CUDA events over `iters` back-to-back refine(steps=2) calls after `warmup`
calls (a refined trajectory stays refined, so every call does the same work), divided by two; the sweep timed the same
way in the same run.  A separate torch.profiler run gives each kernel of a step its time, and for the residual kernel
the HBM bandwidth its byte count implies (per stage knot: the record, z read once with x_{t+1} and lambda_t from the
neighbours' rows in cache, r written) as a fraction of the 3350 GB/s data-sheet peak.  kkt_error is timed the same
two ways: the call (a memset, the residual kernel with one norm per row family, a copy to the host and a synchronise)
from CUDA events, and its kernel from torch.profiler.  Prints one JSON line per config with the card's name and power
limit read in the same run."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_adjoint import card  # noqa: E402

CONFIGS = [("C2", 12, 6, 0, 0, 100, 4096), ("C3", 4, 2, 2, 2, 100, 16384), ("C5", 57, 28, 0, 0, 150, 512)]
MU = 1e-8


def residual_bytes(nx, nu, nc, srec, B, N):
    """HBM bytes of one residual launch over the stage knots (the terminal rows are < 1 % at N >= 100)."""
    z = 2 * nx + nu + nc  # x_t, u_t, v_t, lambda_{t+1}
    return 8 * B * N * (srec + z + z)  # record, z, r


def profiled(torch, f):
    """ms per call of f for each kernel of a refinement step, from torch.profiler (f runs three times)."""
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
        key = ("residual" if "refine_residual" in ev.key else "update" if "linear_step" in ev.key
               else "resolve" if "resolve_kernel" in ev.key else None)
        if key:
            kern[key] = kern.get(key, 0.0) + t / 1e3 / 3
    return kern


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    import aligator_b200.gar as gar
    import bench
    name, power = card()
    for cfg, nx, nu, nc, nct, N, B in CONFIGS:
        stage, term, G0, g0 = bench.synth_batch_torch(torch, B, N, nx, nu, "cuda:0", 7, nc, nct, "control")
        s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nx, N, B)
        s.set_problem(stage, term, G0, g0, memspace=gar.AB2_DEVICE)

        def timed(f):
            for _ in range(args.warmup):
                f()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.iters):
                f()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / args.iters

        sweep_ms = timed(lambda: s.sweep(MU))
        s.sweep(MU)
        k0 = s.kkt_error(MU).max(axis=1)
        norms = s.refine(MU, 2, norms=True)
        k2 = s.kkt_error(MU).max(axis=1)
        step_ms = timed(lambda: s.refine(MU, 2)) / 2
        kkt_ms = timed(lambda: s.kkt_error(MU))
        kkt_kernel_ms = profiled(torch, lambda: s.kkt_error(MU))["residual"]  # the residual kernel's norms
        kern = profiled(torch, lambda: s.refine(MU, 1))
        rb = residual_bytes(nx, nu, nc, s.srec, B, N)
        res_ms = kern.get("residual", float("nan"))
        gbs = rb / (res_ms * 1e-3) / 1e9
        print(json.dumps(dict(config=cfg, batch=B, horizon=N, mu=MU, gpu=name, power_limit=power,
                              sweep_ms=round(sweep_ms, 4), step_ms=round(step_ms, 4),
                              step_over_sweep=round(step_ms / sweep_ms, 2),
                              kernels_ms={k: round(v, 4) for k, v in kern.items()},
                              kkt_error_ms=round(kkt_ms, 4), kkt_error_kernel_ms=round(kkt_kernel_ms, 4),
                              residual_bytes=rb, residual_GBps=round(gbs, 1), residual_frac_of_3350=round(gbs / 3350, 3),
                              kkt_max_unrefined=float(k0.max()), kkt_max_refined=float(k2.max()),
                              norm_first_max=float(norms[:, 0].max()), norm_last_max=float(norms[:, -1].max()))),
              flush=True)
        s.close()


if __name__ == "__main__":
    main()
