"""In-tree build of the CUDA library (sm_90a, H100) -> aligator_b200/libaligator_b200_gar.so.

One object file per compile-time shape of csrc/riccati_configs.h (built in parallel),
plus the C-ABI translation unit, linked with nvcc -shared.  Cross-compiles without a GPU.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import re
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(CSRC, "build")
LIB = os.path.join(PKG, "libaligator_b200_gar.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++"]


def configs():
    txt = open(os.path.join(CSRC, "riccati_configs.h")).read()
    body = txt.split("#else", 1)[1]
    return [tuple(int(v) for v in m.groups())
            for m in re.finditer(r"X\((\d+),\s*(\d+),\s*(\d+),\s*(\d+)\)", body)]


def _digest(paths, extra=""):
    # the compiler flags are part of every object's name: a change of target architecture rebuilds
    h = hashlib.sha256((" ".join(ARCH + FLAGS) + extra).encode())
    for p in paths:
        h.update(open(p, "rb").read())
    return h.hexdigest()[:16]


_INCLUDE = re.compile(r'^\s*#\s*include\s+"([^"]+)"', re.M)


def _sources(src):
    """src and every file it reaches through #include "...", in a fixed order: what an object depends on."""
    seen, todo = set(), [os.path.normpath(src)]
    while todo:
        p = todo.pop()
        if p in seen or not os.path.exists(p):
            continue
        seen.add(p)
        todo += [os.path.normpath(os.path.join(os.path.dirname(p), m)) for m in _INCLUDE.findall(open(p).read())]
    return sorted(seen)


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("build failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
    return r.stdout + r.stderr


def build(verbose=False, force=False, ptxas_v=False):
    os.makedirs(OBJ, exist_ok=True)
    extra = ["-Xptxas", "-v"] if ptxas_v else []
    jobs = []

    def obj(name, src, defines=(), tag=""):
        # the -Xptxas -v flag is part of the digest, so a --ptxas build recompiles and prints every kernel
        src = os.path.join(CSRC, src)
        o = os.path.join(OBJ, "%s_%s.o" % (name, _digest(_sources(src), tag + str(extra))))
        jobs.append((o, [NVCC] + ARCH + FLAGS + extra + list(defines) + ["-c", src, "-o", o]))

    for (nx, nu, nc, g) in configs():
        obj("k_%d_%d_%d" % (nx, nu, nc), "kernel_inst.cu",
            ["-DAB2_NX=%d" % nx, "-DAB2_NU=%d" % nu, "-DAB2_NC=%d" % nc, "-DAB2_G=%d" % g], "%d_%d_%d_%d" % (nx, nu, nc, g))
    for name, src in (("capi", "gar_cuda.cu"), ("block", "block_kernel.cu"),
                      ("assemble", "lq_assemble.cu"), ("adjoint", "lq_adjoint.cu"), ("lq_items", "lq_items.cu"),
                      ("jacobian", "lq_jacobian.cu"), ("refine", "lq_refine.cu"), ("linesearch", "linesearch.cu"),
                      ("inner", "proxddp_inner.cu")):
        obj(name, src)
    todo =[(o, c) for (o, c) in jobs if force or not os.path.exists(o)]
    logs = []
    if todo:
        with cf.ThreadPoolExecutor(max_workers=max(1, min(len(todo), os.cpu_count() or 4))) as ex:
            for out in ex.map(lambda oc: _run(oc[1]), todo):
                logs.append(out)
    objs = [o for (o, _) in jobs]
    stamp = os.path.join(OBJ, "link.stamp")
    want = _digest(objs)
    if force or todo or not os.path.exists(LIB) or not os.path.exists(stamp) or open(stamp).read() != want:
        _run([NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-ccbin", "/usr/bin/g++"])
        open(stamp, "w").write(want)
    # drop stale objects
    keep = set(os.path.basename(o) for o in objs) | {"link.stamp"}
    for f in os.listdir(OBJ):
        if f not in keep:
            os.remove(os.path.join(OBJ, f))
    if verbose:
        print("\n".join(logs))
        print("built", LIB)
    return LIB


if __name__ == "__main__":
    build(verbose=True, force="--force" in sys.argv, ptxas_v="--ptxas" in sys.argv)
