"""Time ab2_gar_tangent against the sweep it is built around, at C2 (nx12 nu6 N100 B4096) and C3 (nx4 nu2 nc2 N100
B16384, mu 1e-3).

    python tools/bench_tangent.py [--iters 50] [--warmup 10]

Per config: the sweep and the whole tangent call, in ms per call from CUDA events over `iters` back-to-back calls
after `warmup` calls; then, from a separate torch.profiler run, each of the tangent call's three kernels with its time
and the HBM bandwidth its byte count implies.  Prints one JSON line per config, with the card's name and power limit
read in the same run."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_adjoint import CONFIGS, card  # noqa: E402


def bytes_per_knot(nx, nu, nc, srec):
    """HBM bytes each streaming kernel of the call moves per stage knot (terminal knots and g0 are < 1 % at N = 100)."""
    vec = nx + nu + nc + nx  # x_t, u_t, v_t, lambda_{t+1}; and the rows of rho
    mat = srec - (2 * nx + nu + nc)  # the matrix part of a record, copied by the records kernel
    return dict(rhs=8 * (srec + 2 * vec), records=8 * (mat + vec + srec))


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
        dot = dict(stage=torch.randn_like(stage), term=torch.randn_like(term), G0=torch.randn_like(G0),
                   g0=torch.randn_like(g0))
        calls = dict(sweep=lambda: s.sweep(mu), tangent=lambda: s.tangent(primal, dot, mu))
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
                calls["tangent"]()
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if ev.device_type.name != "CUDA" or ev.count == 0:
                continue
            t = getattr(ev, "device_time_total", None) or ev.cuda_time_total
            key = ("rhs" if "jacobian_rhs" in ev.key else "records" if "adjoint_records" in ev.key
                   else "sweep" if "kernel" in ev.key and "Memcpy" not in ev.key else None)
            if key:
                kern[key] = kern.get(key, 0.0) + t / ev.count / 1e3  # ms per call
        bpk = bytes_per_knot(nx, nu, nc, s.srec)
        gbs = {k: bpk[k] * B * N / (kern[k] * 1e-3) / 1e9 for k in bpk if kern.get(k)}
        print(json.dumps(dict(config=cfg, batch=B, horizon=N, gpu=name, power_limit=power,
                              sweep_ms=round(ms["sweep"], 4), tangent_ms=round(ms["tangent"], 4),
                              ratio=round(ms["tangent"] / ms["sweep"], 3),
                              kernel_ms={k: round(v, 4) for k, v in kern.items()},
                              kernel_bytes_per_knot=bpk, kernel_GBps={k: round(v, 1) for k, v in gbs.items()},
                              kernel_frac_of_3350={k: round(v / 3350.0, 3) for k, v in gbs.items()})))
        s.close()


if __name__ == "__main__":
    main()
