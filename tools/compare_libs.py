"""Compare two builds of the library bit for bit on the derivative calls of the LQ solve.

    python tools/compare_libs.py OLD.so NEW.so [--out DIR]

Each library runs in its own process (gar.py loads one library per process): on seeded problems at C2, C3 (with
terminal constraints) and C5 shapes, with a scalar and a per-instance mu, after a cycle_append (nonzero ring head), it
calls adjoint, tangent, adjoint_many and tangent_many (nrhs 1 and 8), resolve, refine, refine_many, factor_adjoint and
factor_tangent, with some input and output fields left NULL, and saves every output, including the handle's trajectory
after adjoint and tangent.  The outputs are then compared as uint64 views, so -0.0 and +0.0 differ.  A call a shape
does not support is recorded as refused and must be refused by both.  Prints one JSON line and exits 1 on any
difference."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOL = ("xs", "us", "vs", "vsT", "lam0", "lams")
RHS = ("q", "r", "d", "dN", "g0", "f")
FAC = ("ff", "fb", "vxx", "vx", "fft", "fbt")
# name, (nx, nu, nc, nct, nc0, N, batch)
CASES = [("C2", (12, 6, 0, 0, 12, 20, 48)), ("C3", (4, 2, 2, 2, 4, 20, 96)), ("C5", (57, 28, 0, 0, 57, 5, 3))]


def dump(lib, path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import gen
    import aligator_b200.gar as gar
    gar.LIB_PATH = lib
    res = {}
    for name, (nx, nu, nc, nct, nc0, N, B) in CASES:
        rng = np.random.default_rng(7)
        stage, term, G0, g0 = gar.pack_problems(gen.generate_batch(5, B, N, nx, nu, nc, nct))
        sol = dict(xs=(N + 1, nx), us=(N, nu), vs=(N, nc), vsT=(nct,), lam0=(nc0,), lams=(N, nx))
        dev = lambda a: torch.tensor(np.ascontiguousarray(a), device="cuda")
        rand = lambda *shape: dev(rng.standard_normal(shape))
        nan = lambda *shape: torch.full(shape, float("nan"), dtype=torch.float64, device="cuda")
        for mname, mu in (("scalar", 1e-3), ("vector", rng.uniform(1e-4, 1e-2, B))):
            tag = "%s/%s/" % (name, mname)
            s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
            s.set_problem(stage, term, G0, g0)
            s.sweep(mu)
            s.cycle_append(rng.standard_normal((B, s.srec)) * 0.1 + stage[:, 0])
            rec = dict(stage=(N, s.srec), term=(s.trec,), G0=(nc0 * nx,), g0=(nc0,))

            def keep(key, f):
                try:
                    out = f()
                except gar.GarError as e:
                    res[tag + key + "/refused"] = np.array([1.0])
                    return
                torch.cuda.synchronize()
                for k, v in out.items():
                    res[tag + key + "/" + k] = v.cpu().numpy() if torch.is_tensor(v) else np.asarray(v)

            def traj():
                return {k: s.get(w) for k, w in zip(SOL, (gar.OUT_XS, gar.OUT_US, gar.OUT_VS, gar.OUT_VST,
                                                            gar.OUT_LBD0, gar.OUT_LBDAS))}

            def primal():
                s.sweep(mu)
                return {k: dev(v) for k, v in traj().items()}

            def adjoint():
                g = {k: nan(B, *rec[k]) for k in rec}
                cot = {k: rand(B, *sol[k]) for k in SOL if k != "vs"}  # vs: zero
                s.adjoint(primal(), cot, g, mu)
                return dict(g, **{"w_" + k: v for k, v in traj().items()})

            def tangent():
                s.tangent(primal(), dict(stage=rand(B, *rec["stage"]), G0=rand(B, *rec["G0"]), g0=rand(B, *rec["g0"])),
                          mu)
                return traj()

            keep("adjoint", adjoint)
            keep("tangent", tangent)
            p = primal()
            for R in (1, 8):
                def adjoint_many():
                    g = {k: nan(R, B, *rec[k]) for k in ("stage", "term", "G0")}  # g0 not written
                    w = {k: nan(R, B, *sol[k]) for k in SOL}
                    s.adjoint_many(p, {k: rand(R, B, *sol[k]) for k in SOL if k != "lams"}, w, g, mu)
                    return dict(g, **{"y_" + k: v for k, v in w.items()})

                def tangent_many():
                    w, o = ({k: nan(R, B, *sol[k]) for k in SOL} for _ in range(2))
                    s.tangent_many(p, {k: rand(R, B, *rec[k]) for k in ("stage", "term", "g0")}, w, o, mu)
                    return dict(o, **{"rho_" + k: v for k, v in w.items()})

                keep("adjoint_many%d" % R, adjoint_many)
                keep("tangent_many%d" % R, tangent_many)

            def resolve():
                o = {k: nan(3, B, *sol[k]) for k in SOL}
                s.resolve({k: rand(3, B, *sol[x]) for k, x in zip(RHS, SOL) if k != "f"}, o, mu)
                return o

            def refine_many():
                rhs = {k: rand(2, B, *sol[x]) for k, x in zip(RHS, SOL)}
                z = {k: rand(2, B, *sol[k]) for k in SOL}
                work = {k: nan(2, B, *sol[x]) for k, x in zip(RHS, SOL)}
                work.update({k: nan(2, B, *sol[k]) for k in SOL})
                return dict(z, norms=s.refine_many(rhs, z, work, mu, steps=2, norms=True))

            def factor_adjoint():
                shp = dict(ff=(N, nu + nc + nx), fb=(N, nu + nc + nx, nx), vxx=(N + 1, nx, nx), vx=(N + 1, nx),
                           fft=(nct,), fbt=(nct, nx))
                g = {k: nan(B, *rec[k]) for k in ("stage", "term", "G0")}
                s.factor_adjoint({k: rand(B, *shp[k]) for k in FAC if k != "fbt"}, g, mu)
                return g

            def factor_tangent():
                shp = dict(ff=(N, nu + nc + nx), fb=(N, nu + nc + nx, nx), vxx=(N + 1, nx, nx), vx=(N + 1, nx),
                           fft=(nct,), fbt=(nct, nx))
                o = {k: nan(B, *shp[k]) for k in FAC if k != "fft"}
                s.factor_tangent(dict(stage=rand(B, *rec["stage"]), term=rand(B, *rec["term"])), o, mu)
                return o

            def refine():
                s.sweep(mu)
                n = s.refine(mu, steps=2, norms=True)
                return dict(traj(), norms=n)

            for key, f in (("resolve", resolve), ("refine_many", refine_many), ("factor_adjoint", factor_adjoint),
                           ("factor_tangent", factor_tangent), ("refine", refine)):
                keep(key, f)
            s.close()
    np.savez(path, **res)


def main():
    if sys.argv[1] == "--dump":
        return dump(sys.argv[2], sys.argv[3])
    old, new = sys.argv[1], sys.argv[2]
    out = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else tempfile.mkdtemp()
    os.makedirs(out, exist_ok=True)
    files = []
    for i, lib in enumerate((old, new)):
        f = os.path.join(out, "outputs_%d.npz" % i)
        subprocess.run([sys.executable, os.path.abspath(__file__), "--dump", os.path.abspath(lib), f], check=True)
        files.append(np.load(f))
    a, b = files
    diff = sorted(k for k in set(a.files) | set(b.files)
                  if k not in a.files or k not in b.files or a[k].shape != b[k].shape
                  or not np.array_equal(a[k].view(np.uint64), b[k].view(np.uint64)))
    refused = sorted(k for k in a.files if k.endswith("/refused"))
    detail = {}
    for k in diff:
        if k in a.files and k in b.files and a[k].shape == b[k].shape:
            x, y = a[k].ravel(), b[k].ravel()
            bad = x.view(np.uint64) != y.view(np.uint64)
            ulp = np.abs(x[bad].view(np.int64) - y[bad].view(np.int64))  # exact for same-sign values
            detail[k] = dict(elements=int(bad.sum()), of=int(x.size), max_ulp=int(ulp.max()),
                             max_abs=float(np.abs(x[bad] - y[bad]).max()), max_abs_value=float(np.abs(x).max()))
    print(json.dumps(dict(arrays=len(a.files), doubles=int(sum(a[k].size for k in a.files)), differing=diff,
                          detail=detail, refused=refused)))
    return 1 if diff else 0


if __name__ == "__main__":
    sys.exit(main())
