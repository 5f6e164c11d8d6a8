#!/usr/bin/env python
"""Per-instance scalars against batch-wide ones: the same work with mu / preg / alpha given as [batch] device arrays
(the *_v entry points) or as one number.

  * sweep: ab2_gar_sweep vs ab2_gar_sweep_v at C2, C3 and C4 dimensions;
  * inner: one device inner iteration without model evaluations (multipliers -> assemble -> sweep -> linear_step)
    with scalar or per-instance mu, mu_dyn = 0.1 mu, preg and alpha, at C2 and C3 dimensions.

Each arm is timed with CUDA events over --steps calls after --warmup calls; the two arms alternate --reps times and
the medians are reported with the card's name and power limit.  Needs a CUDA device; prints one JSON line per case."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = {"c2": (12, 6, 0, 0, 100, 4096), "c3": (4, 2, 2, 0, 100, 16384), "c4": (14, 7, 0, 0, 200, 2048)}


def card():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                             "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return torch.cuda.get_device_name(0), pl


def setup(cfg):
    """A handle with a well-posed problem assembled on the device, and the buffers of the inner iteration."""
    import torch
    import aligator_b200.gar as gar
    nx, nu, nc, nct, N, B = CONFIGS[cfg]
    nc0 = nx
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev)
    g.manual_seed(1)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64, device=dev)
    e = lambda *s: torch.empty(*s, dtype=torch.float64, device=dev)
    spd = lambda n, *lead: (lambda M: (M @ M.transpose(-1, -2) / n + torch.eye(n, dtype=torch.float64, device=dev))
                            .reshape(*lead, n * n))(r(*lead, n, n))
    lo = torch.tensor([[float("inf"), -float("inf"), -0.5][i % 3] for i in range(nc)], dtype=torch.float64, device=dev)
    hi = torch.tensor([[float("inf"), 0.0, 0.5][i % 3] for i in range(nc)], dtype=torch.float64, device=dev)
    it = dict(xs=r(B, N + 1, nx), us=r(B, N, nu), vs=r(B, N, nc), vsT=r(B, nct), lam0=r(B, nc0), lams=r(B, N, nx))
    mult_in = dict(xs=it["xs"], lam0=it["lam0"], lams=it["lams"], vs=it["vs"], vsT=it["vsT"], xnext=r(B, N, nx),
                   cval=r(B, N, nc), cval_N=r(B, nct), init_value=r(B, nc0), lo=lo, hi=hi, loN=lo[:nct],
                   hiN=hi[:nct], prev_vs=r(B, N, nc), prev_vsT=r(B, nct))
    mo = dict(slack=e(B, N, nx), lam0_plus=e(B, nc0), lams_plus=e(B, N, nx), vs_plus=e(B, N, nc), vsT_plus=e(B, nct),
              shifted=e(B, N, nc), shifted_N=e(B, nct), Lv=e(B, N, nc), Lv_N=e(B, nct))
    lq = dict(Jx=0.3 * r(B, N, nx * nx), Ju=r(B, N, nx * nu), slack=mo["slack"], Lxx=spd(nx, B, N),
              Lxu=torch.zeros(B, N, nx * nu, dtype=torch.float64, device=dev), Luu=spd(nu, B, N), Lx=r(B, N, nx),
              Lu=r(B, N, nu), cJx=r(B, N, nc * nx), cJu=r(B, N, nc * nu), Lv=mo["Lv"], shifted=mo["shifted"], lo=lo,
              hi=hi, Lxx_N=spd(nx, B), Lx_N=r(B, nx), cJx_N=r(B, nct * nx), Lv_N=mo["Lv_N"],
              shifted_N=mo["shifted_N"], loN=lo[:nct], hiN=hi[:nct], G0=r(B, nc0 * nx), g0=mult_in["init_value"])
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    sc = e(B, 2)
    s.multipliers(mult_in, mo, 1e-3, 1e-4, out=sc)
    s.assemble(lq, 1e-6, 1e3)
    vals = torch.tensor([1e-3, 1e-2, 1e-1], dtype=torch.float64, device=dev)[torch.arange(B, device=dev) % 3]
    per = dict(mu=vals.contiguous(), mu_dyn=(0.1 * vals).contiguous(), preg=(1e-3 * vals).contiguous(),
               mu_inv=(1.0 / vals).contiguous(), alpha=torch.full((B,), 0.5, dtype=torch.float64, device=dev))
    one = dict(mu=1e-2, mu_dyn=1e-3, preg=1e-5, mu_inv=1e2, alpha=0.5)
    trial = {k: torch.empty_like(v) for k, v in it.items()}

    def inner(v):
        s.multipliers(mult_in, mo, v["mu"], v["mu_dyn"], out=sc)
        s.assemble(lq, v["preg"], v["mu_inv"])
        s.sweep(v["mu"])
        s.linear_step(v["alpha"], it, trial)

    return s, per, one, inner


def time_arm(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sweep", default="c2,c3,c4")
    ap.add_argument("--inner", default="c2,c3")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_per_instance needs a CUDA device"
    import __graft_entry__ as g
    g.build()
    name, pl = card()
    cases = [("sweep", c) for c in a.sweep.split(",") if c] + [("inner", c) for c in a.inner.split(",") if c]
    for what, cfg in cases:
        s, per, one, inner = setup(cfg)
        if what == "sweep":
            arms = {"scalar": lambda: s.sweep(one["mu"]), "per_instance": lambda: s.sweep(per["mu"])}
        else:
            arms = {"scalar": lambda: inner(one), "per_instance": lambda: inner(per)}
        ms = {k: [] for k in arms}
        for _ in range(a.reps):  # alternate the arms
            for k, fn in arms.items():
                ms[k].append(time_arm(fn, a.steps, a.warmup))
        med = {k: statistics.median(v) for k, v in ms.items()}
        print(json.dumps(dict(case=what, config=cfg, dims=CONFIGS[cfg], card=name, power_limit=pl,
                              median_ms=med, min_ms={k: min(v) for k, v in ms.items()},
                              max_ms={k: max(v) for k, v in ms.items()},
                              ratio=med["per_instance"] / med["scalar"])), flush=True)
        s.close()


if __name__ == "__main__":
    main()
