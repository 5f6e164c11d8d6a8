"""Time ab2_gar_resolve against the handle's own sweep at C2 (nx12 nu6 N100 B4096), C3 (nx4 nu2 nc2 N100 B16384,
mu 1e-3) and C5 (nx57 nu28 N150 B512), for nrhs in {1, 8, 32}.

    python tools/bench_resolve.py [--iters 50] [--warmup 10]

Per config and nrhs: ms per call from CUDA events over `iters` back-to-back calls after `warmup` calls, the sweep
timed the same way in the same run, the HBM bytes per stage knot the call needs (computed from the shapes) and the
fraction of the 3350 GB/s data-sheet peak those bytes over the call's time imply.  Prints one JSON line each, with the
card's name and power limit read in the same run."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_adjoint import card  # noqa: E402

CONFIGS = [("C2", 12, 6, 0, 0, 100, 4096, 1e-2), ("C3", 4, 2, 2, 2, 100, 16384, 1e-3),
           ("C5", 57, 28, 0, 0, 150, 512, 1e-2)]


def bytes_per_knot(nx, nu, nc, nrhs):
    """HBM bytes per stage knot and instance.  Matrices: A, B, S, R, C, D of the record and V' in the backward pass, FB and
    V' in the forward pass (V' packed).  Per right-hand side: q, r, d, f read twice (backward and vx), the parked
    k, z, a, vx written, then read and rewritten by the forward pass."""
    nr = nu + nc + nx
    P = (nx * (nx + 1) // 2 + 1) & ~1
    mats = nx * nx + 2 * nx * nu + nu * nu + nc * (nx + nu) + nr * nx + 2 * P
    vec = (nx + nu + nc + nx) * 2 + 3 * (nu + nc + 2 * nx)
    return dict(matrices=8 * mats, per_rhs=8 * vec, total=8 * (mats + nrhs * vec))


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
        shapes = dict(q=(B, N + 1, nx), r=(B, N, nu), d=(B, N, nc), dN=(B, nct), g0=(B, nx), f=(B, N, nx))
        sol = dict(xs=shapes["q"], us=shapes["r"], vs=shapes["d"], vsT=shapes["dN"], lam0=shapes["g0"],
                   lams=shapes["f"])

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

        sweep_ms = timed(lambda: s.sweep(mu))
        for nrhs in (1, 8, 32):
            h = {k: torch.randn((nrhs,) + sh, dtype=torch.float64, device="cuda") for k, sh in shapes.items()}
            out = {k: torch.empty((nrhs,) + sh, dtype=torch.float64, device="cuda") for k, sh in sol.items()}
            ms = timed(lambda: s.resolve(h, out, mu))
            bpk = bytes_per_knot(nx, nu, nc, nrhs)
            gbs = bpk["total"] * B * N / (ms * 1e-3) / 1e9
            print(json.dumps(dict(config=cfg, batch=B, horizon=N, nrhs=nrhs, gpu=name, power_limit=power,
                                  sweep_ms=round(sweep_ms, 4), resolve_ms=round(ms, 4),
                                  resolve_over_sweep=round(ms / sweep_ms, 3),
                                  ms_per_rhs=round(ms / nrhs, 4), bytes_per_knot=bpk, GBps=round(gbs, 1),
                                  frac_of_3350=round(gbs / 3350.0, 3))), flush=True)
        s.close()


if __name__ == "__main__":
    main()
