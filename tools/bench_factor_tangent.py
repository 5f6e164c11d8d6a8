"""Time ab2_gar_factor_tangent against the handle's own sweep and ab2_gar_factor_adjoint at C2 (nx12 nu6 N100 B4096),
C3 (nx4 nu2 nc2 nct2 N100 B16384, mu 1e-3) and C5 (nx57 nu28 N150 B512), with every tangent field given and with the
A and B blocks alone.

    python tools/bench_factor_tangent.py [--iters 30] [--warmup 5]

Per config and tangent set: ms per call from CUDA events over `iters` back-to-back calls after `warmup` calls, the
sweep and factor_adjoint (every cotangent field given) timed the same way in the same run, the HBM bytes per stage knot
the call needs (computed from the shapes) and the fraction of the 3350 GB/s data-sheet peak those bytes over the call's
time imply.  Prints one JSON line each, with the card's name and power limit read in the same run."""
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


def bytes_per_knot(nx, nu, nc, all_fields, packed):
    """HBM bytes per stage knot and instance.  Reads: A, B, f, S, R, C, D of the record, V' (packed lower triangle on
    the warp kernel, else full), the K and Z rows of FB, k and z of FF, vx; the tangent record (all of it, or A and B
    alone); writes: the FF, FB, VXX (full) and VX tangents."""
    n, nr = nu + nc, nu + nc + nx
    P = (nx * (nx + 1) // 2 + 1) & ~1 if packed else nx * nx
    srec = 2 * nx * nx + 2 * nx * nu + nu * nu + 2 * nx + nu + nc * (nx + nu + 1)
    srec += srec % 2
    reads = nx * nx + 2 * nx * nu + nx + nu * nu + nc * (nx + nu) + P + n * nx + n + nx
    dot = srec if all_fields else nx * nx + nx * nu
    writes = nr + nr * nx + nx * nx + nx
    return dict(reads=8 * reads, tangent=8 * dot, writes=8 * writes, total=8 * (reads + dot + writes))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
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
        nr = nu + nc + nx
        shapes = dict(ff=(B, N, nr), fb=(B, N, nr * nx), vxx=(B, N + 1, nx * nx), vx=(B, N + 1, nx), fft=(B, nct),
                      fbt=(B, nct * nx))
        out = {k: torch.empty(v, dtype=torch.float64, device="cuda") for k, v in shapes.items()}
        cot = {k: torch.randn(v, dtype=torch.float64, device="cuda") for k, v in shapes.items()}
        grad = dict(stage=torch.empty_like(stage), term=torch.empty_like(term))
        dot_all = dict(stage=torch.randn_like(stage), term=torch.randn_like(term))
        dot_ab = dict(stage=torch.zeros_like(stage))
        dot_ab["stage"][..., :nx * nx + nx * nu] = torch.randn_like(dot_ab["stage"][..., :nx * nx + nx * nu])

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
        s.backward(mu)
        adj_ms = timed(lambda: s.factor_adjoint(cot, grad, mu))
        packed = gar.supported(nx, nu, nc, nx) == 1  # the warp-per-instance sweep leaves Vxx packed
        for fields, d in (("all", dot_all), ("AB", dot_ab)):
            ms = timed(lambda: s.factor_tangent(d, out, mu))
            bpk = bytes_per_knot(nx, nu, nc, fields == "all", packed)
            gbs = bpk["total"] * B * N / (ms * 1e-3) / 1e9
            print(json.dumps(dict(config=cfg, batch=B, horizon=N, tangents=fields, gpu=name, power_limit=power,
                                  sweep_ms=round(sweep_ms, 4), factor_adjoint_ms=round(adj_ms, 4),
                                  factor_tangent_ms=round(ms, 4), over_sweep=round(ms / sweep_ms, 3),
                                  over_factor_adjoint=round(ms / adj_ms, 3), bytes_per_knot=bpk, GBps=round(gbs, 1),
                                  frac_of_3350=round(gbs / 3350.0, 3))), flush=True)
        s.close()


if __name__ == "__main__":
    main()
