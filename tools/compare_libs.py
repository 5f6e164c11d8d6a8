"""Compare two builds of the library bit for bit on the derivative calls of the LQ solve.

    python tools/compare_libs.py OLD.so NEW.so [--out DIR]

Each library runs in its own process (gar.py loads one library per process): on seeded problems at C2, C3 (with
terminal constraints) and C5 shapes, with a scalar and a per-instance mu, after a cycle_append (nonzero ring head), it
calls adjoint, tangent, adjoint_many and tangent_many (nrhs 1 and 8), resolve (nrhs 3 and 33), refine, refine_many,
factor_adjoint and factor_tangent, with some input and output fields left NULL, and saves every output, including the
handle's trajectory after adjoint and tangent.  On parametric handles at C2 and C3 shapes it calls theta_tangent and
theta_adjoint at nrhs 1, 8 and 33 (33 spans two chunks of directions).  The outputs are then compared as uint64 views, so -0.0 and +0.0 differ.  A call a shape
does not support is recorded as refused and must be refused by both.

It also records a state transcript for each handle kind (warp kernel at C2, CTA kernel at C5, dense, parallel with two
legs, parametric): a fixed script of state-changing calls, each followed by every call the handle's state gates, and
after every call its return code and message, the launch-count delta, factor_epoch and the ring heads.  The
transcripts must be equal.  Prints one JSON line and exits 1 on any difference."""
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
# parametric handles for the theta calls: name, (nx, nu, nc, nct, nc0, nth, N, batch)
THETA_CASES = [("C2_nth4", (12, 6, 0, 0, 12, 4, 20, 48)), ("C3_nth2", (4, 2, 2, 2, 4, 2, 20, 96))]
# the state transcript's handle kinds: name, handle options, (nx, nu, N, batch) with nc = nct = 0 and nc0 = nx
KINDS = [("warp_C2", {}, (12, 6, 6, 8)), ("cta_C5", {}, (57, 28, 3, 2)), ("dense", dict(dense=True), (12, 6, 6, 8)),
         ("legs2", dict(legs=2), (12, 6, 6, 8)), ("parametric", dict(nth=2), (12, 6, 6, 8))]


def transcript(gar, torch, kw, dims):
    """One line per call of the script: name, return code and message, launch-count delta, factor_epoch, ring heads."""
    import ctypes as C
    import gen
    from inner_cases import random_fddp
    nx, nu, N, B = dims
    rng = np.random.default_rng(11)
    s = gar.CudaRiccatiBatch(nx, nu, 0, 0, nx, N, B, **kw)
    plain = gar.pack_problems(gen.generate_batch(3, B, N, nx, nu, 0, 0))
    stage, term = np.zeros((B, N, s.srec)), np.zeros((B, s.trec))  # (parametric records: a zero parameter tail)
    stage[..., :plain[0].shape[-1]], term[:, :plain[1].shape[-1]] = plain[0], plain[1]
    G0, g0 = plain[2], plain[3]
    dev = lambda a: torch.tensor(np.ascontiguousarray(a), device="cuda")
    zeros = lambda *shape: torch.zeros(shape, dtype=torch.float64, device="cuda")
    sol = dict(xs=(B, N + 1, nx), us=(B, N, nu), vs=(B, N, 0), vsT=(B, 0), lam0=(B, nx), lams=(B, N, nx))
    rec = dict(stage=(B, N, s.srec), term=(B, s.trec), G0=(B, nx * nx), g0=(B, nx))
    cm = lambda a: np.ascontiguousarray(np.swapaxes(a, -1, -2))
    fd = random_fddp(rng, B, N, nx, nu)
    fddp = {k: dev(cm(v) if v.ndim >= 3 and k not in ("fs", "Lx", "Lu", "Lx_N") else v) for k, v in fd.items()}
    lq = {k: fddp[k] for k in ("Jx", "Ju", "Lxx", "Lxu", "Luu", "Lx", "Lu", "Lxx_N", "Lx_N")}
    lq.update(slack=fddp["fs"][:, 1:].contiguous(), G0=dev(np.tile(-np.eye(nx).ravel(), (B, 1))),
              g0=fddp["fs"][:, 0].contiguous())
    new_last = stage[:, 0] + 0.01
    mu = 1e-3
    sweep_out = {gar.OUT_XS: np.empty(B * (N + 1) * nx), gar.OUT_VXX: np.empty(B * (N + 1) * nx * nx)}
    gated = [
        ("resolve", lambda: s.resolve({}, {k: zeros(1, *v) for k, v in sol.items()}, mu)),
        ("refine", lambda: s.refine(mu, 1)),
        ("factor_adjoint", lambda: s.factor_adjoint({}, {k: zeros(*v) for k, v in rec.items()}, mu)),
        ("kkt_error", lambda: s.kkt_error(mu)),
        ("first_step_policy", lambda: s.first_step_policy_into(zeros(B, nu, nx + 1))),
        ("get_gains", lambda: s.get_gains()),
    ]
    primal = lambda: {k: zeros(*v) for k, v in sol.items()}
    script = [
        ("set_problem", lambda: s.set_problem(stage, term, G0, g0)),
        ("forward", lambda: s.forward()),
        ("backward", lambda: s.backward(mu)),
        ("forward", lambda: s.forward()),
        ("adjoint", lambda: s.adjoint(primal(), {}, {}, mu)),
        ("forward", lambda: s.forward()),
        ("tangent", lambda: s.tangent(primal(), {}, mu)),
        ("sweep", lambda: s.sweep(mu)),
        ("cycle_append", lambda: s.cycle_append(new_last)),
        ("forward", lambda: s.forward()),
        ("sweep", lambda: s.sweep(np.full(B, mu))),
        ("set_problem", lambda: s.set_problem(None, term)),
        ("backward", lambda: s.backward(mu)),
        ("assemble", lambda: s.assemble(lq, 1e-4, 1.0)),
        ("sweep", lambda: s.sweep(mu)),
        ("sweep_host", lambda: (s.sweep_host(stage, term, G0, g0, mu, sweep_out), s.synchronize())),
        ("cycle_append", lambda: s.cycle_append(new_last)),
        ("fddp_backward_pass", lambda: s.fddp_backward_pass(fddp, 1e-4)),
    ]
    lines = []
    for name, f in [(n, f) for step in script for n, f in [step] + gated]:
        torch.cuda.synchronize()
        n0 = s.launch_count()
        try:
            f()
            err = "0"
        except gar.GarError as e:
            err = str(e)
        torch.cuda.synchronize()
        fh, sh = C.c_int(), C.c_int()
        gar.lib().ab2_gar_ring_heads(s.h, C.byref(fh), C.byref(sh))
        lines.append("%s: %s | launches +%d | epoch %d | heads %d %d"
                     % (name, err, s.launch_count() - n0, s.factor_epoch(), fh.value, sh.value))
    s.close()
    return lines


def dump(lib, path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import gen
    import lq_cases
    import aligator_b200.gar as gar
    gar.LIB_PATH = lib
    res = {}
    dev = lambda a: torch.tensor(np.ascontiguousarray(a), device="cuda")
    rand = lambda *shape: dev(rng.standard_normal(shape))
    nan = lambda *shape: torch.full(shape, float("nan"), dtype=torch.float64, device="cuda")

    def keep(key, f):
        """f()'s outputs under tag/key/..., or tag/key/refused"""
        try:
            out = f()
        except gar.GarError as e:
            res[tag + key + "/refused"] = np.array([1.0])
            return
        torch.cuda.synchronize()
        for k, v in out.items():
            res[tag + key + "/" + k] = v.cpu().numpy() if torch.is_tensor(v) else np.asarray(v)

    for name, (nx, nu, nc, nct, nc0, N, B) in CASES:
        rng = np.random.default_rng(7)
        stage, term, G0, g0 = gar.pack_problems(gen.generate_batch(5, B, N, nx, nu, nc, nct))
        sol = dict(xs=(N + 1, nx), us=(N, nu), vs=(N, nc), vsT=(nct,), lam0=(nc0,), lams=(N, nx))
        for mname, mu in (("scalar", 1e-3), ("vector", rng.uniform(1e-4, 1e-2, B))):
            tag = "%s/%s/" % (name, mname)
            s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B)
            s.set_problem(stage, term, G0, g0)
            s.sweep(mu)
            s.cycle_append(rng.standard_normal((B, s.srec)) * 0.1 + stage[:, 0])
            rec = dict(stage=(N, s.srec), term=(s.trec,), G0=(nc0 * nx,), g0=(nc0,))

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

            def resolve(R):
                o = {k: nan(R, B, *sol[k]) for k in SOL}
                s.resolve({k: rand(R, B, *sol[x]) for k, x in zip(RHS, SOL) if k != "f"}, o, mu)
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

            for key, f in (("resolve", lambda: resolve(3)), ("resolve33", lambda: resolve(33)),
                           ("refine_many", refine_many), ("factor_adjoint", factor_adjoint),
                           ("factor_tangent", factor_tangent), ("refine", refine)):
                keep(key, f)
            s.close()
    for name, (nx, nu, nc, nct, nc0, nth, N, B) in THETA_CASES:
        rng = np.random.default_rng(9)
        tag = name + "/"
        sol = dict(xs=(N + 1, nx), us=(N, nu), vs=(N, nc), vsT=(nct,), lam0=(nc0,), lams=(N, nx))
        s = gar.CudaRiccatiBatch(nx, nu, nc, nct, nc0, N, B, nth=nth)
        s.set_problem(*gar.pack_problems([lq_cases.make_problem([5, b], N, nx, nu, nc, nct, nth, gv=True)
                                          for b in range(B)]))
        s.backward(1e-3)
        s.forward(theta=rng.standard_normal((B, nth)))
        for R in (1, 8, 33):
            def theta_tangent():
                o = {k: nan(R, B, *sol[k]) for k in SOL}
                s.theta_tangent(rand(R, B, nth), o)
                return o

            def theta_adjoint():
                tb = nan(R, B, nth)
                s.theta_adjoint({k: rand(R, B, *sol[k]) for k in SOL if k != "us"}, tb)  # us: zero
                return dict(theta_bar=tb)

            keep("theta_tangent%d" % R, theta_tangent)
            keep("theta_adjoint%d" % R, theta_adjoint)
        s.close()
    for name, kw, dims in KINDS:
        res["transcript/" + name] = np.array(transcript(gar, torch, kw, dims))
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
    same = lambda x, y: np.array_equal(x, y) if x.dtype.kind == "U" else np.array_equal(x.view(np.uint64),
                                                                                         y.view(np.uint64))
    diff = sorted(k for k in set(a.files) | set(b.files)
                  if k not in a.files or k not in b.files or a[k].shape != b[k].shape or not same(a[k], b[k]))
    refused = sorted(k for k in a.files if k.endswith("/refused"))
    detail = {}
    for k in diff:
        if k.startswith("transcript/") and k in a.files and k in b.files and a[k].shape == b[k].shape:
            detail[k] = [dict(old=x, new=y) for x, y in zip(a[k].tolist(), b[k].tolist()) if x != y][:5]
        elif k in a.files and k in b.files and a[k].shape == b[k].shape:
            x, y = a[k].ravel(), b[k].ravel()
            bad = x.view(np.uint64) != y.view(np.uint64)
            ulp = np.abs(x[bad].view(np.int64) - y[bad].view(np.int64))  # exact for same-sign values
            detail[k] = dict(elements=int(bad.sum()), of=int(x.size), max_ulp=int(ulp.max()),
                             max_abs=float(np.abs(x[bad] - y[bad]).max()), max_abs_value=float(np.abs(x).max()))
    transcripts = {k: len(a[k]) for k in a.files if k.startswith("transcript/")}
    print(json.dumps(dict(arrays=len(a.files), doubles=int(sum(a[k].size for k in a.files if a[k].dtype.kind == "f")),
                          differing=diff, detail=detail, refused=refused, transcript_lines=transcripts)))
    return 1 if diff else 0


if __name__ == "__main__":
    sys.exit(main())
