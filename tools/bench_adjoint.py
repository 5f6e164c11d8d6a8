"""Time ab2_gar_adjoint against the sweep it is built around, at C2 (nx12 nu6 N100 B4096) and C3 (nx4 nu2 nc2 N100
B16384, mu 1e-3).

    python tools/bench_adjoint.py [--iters 50] [--warmup 10]

Per config: the sweep and the whole adjoint call, in ms per call from CUDA events over `iters` back-to-back calls
after `warmup` calls; then, from one torch.profiler run, each of the adjoint call's three kernels with its time and
the HBM bandwidth its byte count implies.  Prints one JSON line per config, with the card's name and power limit
read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = [("C2", 12, 6, 0, 0, 100, 4096, 1e-2), ("C3", 4, 2, 2, 0, 100, 16384, 1e-3)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")[:2]]
        return name, power
    except Exception as e:  # the numbers are still printed, without the card's identity
        return "unknown (%s)" % e, "unknown"


def bytes_per_knot(nx, nu, nc, srec):
    """HBM bytes each kernel of the call moves per stage knot (terminal knots and g0 are < 1 % at N = 100)."""
    vec = nx + nu + nc + nx  # x_t, u_t, v_t, lambda_{t+1}
    mat = srec - (2 * nx + nu + nc)  # the matrix part of a record, copied
    return dict(records=8 * (mat + vec + srec), grad=8 * (2 * vec + srec))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    import aligator_b200.gar as gar
    import bench
    name, power = card()
    for cfg, nx, nu, nc, nct, N, B, mu in CONFIGS:
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
        cot = {k: torch.randn_like(v) for k, v in primal.items()}
        grad = dict(stage=torch.empty_like(stage), term=torch.empty_like(term), G0=torch.empty_like(G0),
                    g0=torch.empty_like(g0))
        calls = dict(sweep=lambda: s.sweep(mu), adjoint=lambda: s.adjoint(primal, cot, grad, mu))
        ms = {}
        for k, f in calls.items():
            for _ in range(args.warmup):
                f()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.iters):
                f()
            e1.record()
            torch.cuda.synchronize()
            ms[k] = e0.elapsed_time(e1) / args.iters
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                calls["adjoint"]()
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if ev.device_type.name != "CUDA" or ev.count == 0:
                continue
            t = getattr(ev, "device_time_total", None) or ev.cuda_time_total
            key = ("records" if "adjoint_records" in ev.key else "grad" if "jacobian_grad" in ev.key
                   else "sweep" if "kernel" in ev.key and "Memcpy" not in ev.key else None)
            if key:
                kern[key] = kern.get(key, 0.0) + t / ev.count / 1e3  # ms per call
        bpk = bytes_per_knot(nx, nu, nc, s.srec)
        gbs = {k: bpk[k] * B * N / (kern[k] * 1e-3) / 1e9 for k in bpk if kern.get(k)}
        print(json.dumps(dict(config=cfg, batch=B, horizon=N, gpu=name, power_limit=power,
                              sweep_ms=round(ms["sweep"], 4), adjoint_ms=round(ms["adjoint"], 4),
                              ratio=round(ms["adjoint"] / ms["sweep"], 3),
                              kernel_ms={k: round(v, 4) for k, v in kern.items()},
                              kernel_bytes_per_knot=bpk, kernel_GBps={k: round(v, 1) for k, v in gbs.items()})))
        s.close()


if __name__ == "__main__":
    main()
