"""Time the theta derivatives of parametric handles (ab2_gar_theta_tangent, ab2_gar_theta_adjoint) at C2 dimensions
(nx12 nu6 N100 B4096) with nth in {1, 4, 12} and C3 dimensions (nx4 nu2 nc2 nct2 N100 B16384, mu 1e-3) with nth 2.

    python tools/bench_theta.py [--iters 30] [--warmup 5]

Per config, ms per call from CUDA events over `iters` back-to-back calls after `warmup` calls, all in one run:
  sweep      backward + forward_theta (what the solve costs)
  tangent    theta_tangent at nrhs = nth: the whole Jacobian J
  adjoint    theta_adjoint at nrhs = 1: one gradient J^T zbar
  fwd_diff   nth + 1 forward_theta calls: the Jacobian by differences, as a user does without these calls
and, for tangent and adjoint, the HBM bytes the algorithm needs (computed from the shapes below: per stage knot and
instance FB, FTH, Vxx and Vxt read once, 8 (nr nx + nr nth + nx^2 + nx nth) bytes, plus the per-direction vectors)
and the fraction of the 3350 GB/s data-sheet peak those bytes over the call's time imply.  The problems are 8 seeded
parametric instances tiled over the batch.  One JSON line per config, with the card's name and power limit read in
the same run."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_adjoint import card  # noqa: E402

# name, nx, nu, nc, nct, nth, N, B, mu
CONFIGS = [("C2", 12, 6, 0, 0, 1, 100, 4096, 1e-8), ("C2", 12, 6, 0, 0, 4, 100, 4096, 1e-8),
           ("C2", 12, 6, 0, 0, 12, 100, 4096, 1e-8), ("C3", 4, 2, 2, 2, 2, 100, 16384, 1e-3)]


def algorithmic_bytes(nx, nu, nc, nct, nc0, nth, N, B, nrhs, adjoint):
    """HBM bytes of one call: per instance and stage knot the matrices FB, FTH, Vxx, Vxt once (one item holds all
    nrhs <= 32 directions), and per direction and knot the vectors written (tangent: u, v, x, lambda) or read
    (adjoint: their cotangents); the initial and terminal blocks and theta itself are left out (under 2 % here)."""
    nr = nu + nc + nx
    mats = nr * nx + nr * nth + nx * nx + nx * nth
    vec = nu + nc + 2 * nx
    return 8 * B * N * (mats + nrhs * vec)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    import torch
    import __graft_entry__ as g
    g.build()
    import aligator_b200.gar as gar
    import lq_cases
    name, power = card()

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

    for cfg, nx, nu, nc, nct, nth, N, B, mu in CONFIGS:
        probs = [lq_cases.make_problem([91, b], N, nx, nu, nc, nct, nth) for b in range(8)]
        recs = [np.ascontiguousarray(np.concatenate([r] * (B // 8))) for r in gar.pack_problems(probs)]
        s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nx, N, B, nth=nth)
        s.set_problem(*[torch.from_numpy(r).cuda() for r in recs], memspace=gar.AB2_DEVICE)
        theta = torch.randn((B, nth), dtype=torch.float64, device="cuda")

        def sweep():
            s.backward(mu)
            s.forward(theta=theta)

        sweep()
        torch.cuda.synchronize()
        assert np.all(s.status() == 0)
        shapes = dict(xs=(B, N + 1, nx), us=(B, N, nu), vs=(B, N, nc), vsT=(B, nct), lam0=(B, nx), lams=(B, N, nx))
        dth = torch.randn((nth, B, nth), dtype=torch.float64, device="cuda")
        out = {k: torch.empty((nth,) + sh, dtype=torch.float64, device="cuda") for k, sh in shapes.items()}
        cot = {k: torch.randn((1,) + sh, dtype=torch.float64, device="cuda") for k, sh in shapes.items()}
        tb = torch.empty((1, B, nth), dtype=torch.float64, device="cuda")
        sweep_ms = timed(sweep)
        tan_ms = timed(lambda: s.theta_tangent(dth, out))
        adj_ms = timed(lambda: s.theta_adjoint(cot, tb))

        def fwd_diff():
            for _ in range(nth + 1):
                s.forward(theta=theta)

        diff_ms = timed(fwd_diff)
        row = dict(config=cfg, nx=nx, nu=nu, nc=nc, nct=nct, nth=nth, horizon=N, batch=B, gpu=name, power_limit=power,
                   sweep_ms=round(sweep_ms, 4), fwd_diff_ms=round(diff_ms, 4))
        for key, ms, nrhs, adj in (("tangent", tan_ms, nth, False), ("adjoint", adj_ms, 1, True)):
            by = algorithmic_bytes(nx, nu, nc, nct, nx, nth, N, B, nrhs, adj)
            gbs = by / (ms * 1e-3) / 1e9
            row.update({key + "_nrhs": nrhs, key + "_ms": round(ms, 4), key + "_bytes": by, key + "_GBps": round(gbs, 1),
                        key + "_frac_of_3350": round(gbs / 3350.0, 3)})
        row["jacobian_speedup_vs_fwd_diff"] = round(diff_ms / tan_ms, 2)
        print(json.dumps(row), flush=True)
        s.close()


if __name__ == "__main__":
    main()
