#!/usr/bin/env python
"""Timings of the inner-iteration kernels (ab2_gar_multipliers, ab2_gar_lagrangian_gradient, ab2_gar_criterion) at
BASELINE config 2 and 3 dims, and of one device-resident inner iteration without model evaluations.

Per kernel: CUDA-event time over --launches launches after warm-up, the algorithmic bytes (every input array read
once, every output written once, counted from the shapes below), GB/s and the fraction of the H100 SXM data sheet's
3350 GB/s.  Then the chain multipliers -> al_value -> lagrangian_gradient -> criterion -> assemble -> sweep ->
lagrangian_gradient(plus) -> directional_derivative -> linear_step -> multipliers -> al_value against the shorter
chain bench.py's e2e_device times (assemble -> sweep -> linear_step -> directional_derivative), both wall-clock per
iteration with the host waiting for the [batch] scalars at the end, as a line search would.
Needs a CUDA device; prints one JSON line per config."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_GBS = 3350.0  # H100 SXM data sheet HBM3 bandwidth
CONFIGS = {"c2": (12, 6, 0, 0, 100, 4096), "c3": (4, 2, 2, 0, 100, 16384)}  # nx, nu, nc, nct, N, batch (nc0 = nx)


def algorithmic_bytes(nx, nu, nc, nct, nc0, N, B):
    """Doubles each kernel must move at least once, times 8."""
    mult = (2 * nc0 + 3 * N * nx + 3 * N * nc + 3 * nct          # init_value, lam0; xnext, xs[1..N], lams; cval, prev, vs
            + nc0 + 2 * N * nx + 3 * N * nc + 3 * nct + 2)       # lam0_plus; slack, lams_plus; shifted, Lv, vs_plus; scalars
    grad = (N * (nx + nu) + nx                                    # lx, lu, lx_N
            + N * (nx * nx + nx * nu) + N * nc * (nx + nu) + nct * nx + nc0 * nx   # Jx, Ju, cJx, cJu, cJx_N, G0
            + nc0 + N * nx + N * nc + nct                         # lam0, lams, vs, vsT
            + (N + 1) * nx + N * nu)                              # Lx, Lx_N, Lu
    crit = (N + 1) * nx + N * nu + nc0 + max(N - 1, 0) * nx + N * nc + nct + 2
    return {k: 8 * B * v for k, v in dict(multipliers=mult, lagrangian_gradient=grad, criterion=crit).items()}


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                             "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def run(cfg, launches, iters):
    import torch
    import aligator_b200.gar as gar
    nx, nu, nc, nct, N, B = CONFIGS[cfg]
    nc0 = nx
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev)
    g.manual_seed(1)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64, device=dev)
    e = lambda *s: torch.empty(*s, dtype=torch.float64, device=dev)
    mu, mu_dyn = 1e-3, 1e-3
    lo = torch.tensor([[float("inf"), -float("inf"), -0.5][i % 3] for i in range(nc)], dtype=torch.float64, device=dev)
    hi = torch.tensor([[float("inf"), 0.0, 0.5][i % 3] for i in range(nc)], dtype=torch.float64, device=dev)
    it = dict(xs=r(B, N + 1, nx), us=r(B, N, nu), vs=r(B, N, nc), vsT=r(B, nct), lam0=r(B, nc0), lams=r(B, N, nx))
    model = dict(xnext=r(B, N, nx), cval=r(B, N, nc), cval_N=r(B, nct), init_value=r(B, nc0), lx=r(B, N, nx),
                 lu=r(B, N, nu), lx_N=r(B, nx), Jx=r(B, N, nx * nx), Ju=r(B, N, nx * nu), cJx=r(B, N, nc * nx),
                 cJu=r(B, N, nc * nu), cJx_N=r(B, nct * nx), G0=r(B, nc0 * nx), Lxx=r(B, N, nx * nx),
                 Lxu=r(B, N, nx * nu), Luu=r(B, N, nu * nu), Lxx_N=r(B, nx * nx), cost=r(B))
    for k in ("Lxx", "Luu", "Lxx_N"):  # well-posed sweeps: symmetric positive definite Hessians
        n = {"Luu": nu}.get(k, nx)
        M = model[k].view(*model[k].shape[:-1], n, n)
        model[k] = (M @ M.transpose(-1, -2) / n + torch.eye(n, dtype=torch.float64, device=dev)).reshape(model[k].shape)
    prev = dict(prev_vs=r(B, N, nc), prev_vsT=r(B, nct))
    s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
    mo = dict(slack=e(B, N, nx), lam0_plus=e(B, nc0), lams_plus=e(B, N, nx), vs_plus=e(B, N, nc), vsT_plus=e(B, nct),
              shifted=e(B, N, nc), shifted_N=e(B, nct), Lv=e(B, N, nc), Lv_N=e(B, nct))
    sc = e(B, 2)
    g1 = dict(Lx=e(B, N, nx), Lx_N=e(B, nx), Lu=e(B, N, nu), Lxs=e(B, N + 1, nx), Lus=e(B, N, nu))
    g2 = dict(Lxs=e(B, N + 1, nx), Lus=e(B, N, nu))
    mult_in = dict(xs=it["xs"], lam0=it["lam0"], lams=it["lams"], vs=it["vs"], vsT=it["vsT"], xnext=model["xnext"],
                   cval=model["cval"], cval_N=model["cval_N"], init_value=model["init_value"], lo=lo, hi=hi,
                   loN=lo[:nct], hiN=hi[:nct], **prev)
    lag = lambda mult: dict(lx=model["lx"], lu=model["lu"], lx_N=model["lx_N"], Jx=model["Jx"], Ju=model["Ju"],
                            cJx=model["cJx"], cJu=model["cJu"], cJx_N=model["cJx_N"], G0=model["G0"], **mult)
    lag_it = lag(dict(lam0=it["lam0"], lams=it["lams"], vs=it["vs"], vsT=it["vsT"]))
    plus = dict(lam0=mo["lam0_plus"], lams=mo["lams_plus"], vs=mo["vs_plus"], vsT=mo["vsT_plus"])
    lag_plus = lag(plus)
    crit_in = dict(Lxs=g1["Lxs"], Lus=g1["Lus"], init_value=model["init_value"], slack=mo["slack"], Lv=mo["Lv"],
                   Lv_N=mo["Lv_N"])
    lag_assemble_out = {k: g1[k] for k in ("Lx", "Lx_N", "Lu")}
    kernels = {
        "multipliers": lambda: s.multipliers(mult_in, mo, mu, mu_dyn, out=sc),
        "lagrangian_gradient": lambda: s.lagrangian_gradient(lag_it, lag_assemble_out),
        "criterion": lambda: s.criterion(crit_in, out=sc),
    }
    nbytes = algorithmic_bytes(nx, nu, nc, nct, nc0, N, B)
    res = {}
    for name, fn in kernels.items():
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / launches
        gbs = nbytes[name] / (ms * 1e-3) / 1e9
        res[name] = {"ms": ms, "bytes": nbytes[name], "GB_per_s": gbs, "frac_of_3350": gbs / PEAK_GBS}

    lq = dict(Jx=model["Jx"], Ju=model["Ju"], slack=mo["slack"], Lxx=model["Lxx"], Lxu=model["Lxu"], Luu=model["Luu"],
              Lx=g1["Lx"], Lu=g1["Lu"], cJx=model["cJx"], cJu=model["cJu"], Lv=mo["Lv"], shifted=mo["shifted"],
              lo=lo, hi=hi, Lxx_N=model["Lxx_N"], Lx_N=g1["Lx_N"], cJx_N=model["cJx_N"], Lv_N=mo["Lv_N"],
              shifted_N=mo["shifted_N"], loN=lo[:nct], hiN=hi[:nct], G0=model["G0"], g0=model["init_value"])
    trial = {k: torch.empty_like(v) for k, v in it.items()}

    def inner_iteration():
        s.multipliers(mult_in, mo, mu, mu_dyn, out=sc)
        s.al_value(plus, model["cost"], mu_dyn, mu)                            # phi0 (host)
        s.lagrangian_gradient(lag_it, g1)
        s.criterion(crit_in, out=sc)
        s.assemble(lq, 1e-8, 1.0 / mu)
        s.sweep(mu)
        s.lagrangian_gradient(lag_plus, g2)
        s.directional_derivative(g2["Lxs"], g2["Lus"])                          # dphi0 (host)
        s.linear_step(1.0, it, trial)
        s.multipliers(dict(mult_in, xs=trial["xs"], lam0=trial["lam0"], lams=trial["lams"], vs=trial["vs"],
                           vsT=trial["vsT"]), mo, mu, mu_dyn, out=sc)
        return s.al_value(plus, model["cost"], mu_dyn, mu)                     # phi(1) (host)

    def e2e_device():  # bench.py's chain, with the Lagrangian gradients taken as given
        s.assemble(lq, 1e-8, 1.0 / mu)
        s.sweep(mu)
        s.linear_step(1.0, it, trial)
        return s.directional_derivative(g2["Lxs"], g2["Lus"])

    chains = {}
    for name, fn in (("inner_iteration", inner_iteration), ("e2e_device", e2e_device)):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
        chains[name] = {"ms_per_iteration": (time.perf_counter() - t0) / iters * 1e3}
    s.close()
    return {"config": cfg, "dims": dict(nx=nx, nu=nu, nc=nc, nct=nct, nc0=nc0, horizon=N, batch=B), "kernels": res,
            "chains": chains}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c2,c3")
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_inner.py needs a CUDA device")
    import __graft_entry__ as g
    g.build()
    name, pl = card()
    for cfg in a.configs.split(","):
        out = run(cfg, a.launches, a.iters)
        out.update(card=name, power_limit=pl)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
