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


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("build failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
    return r.stdout + r.stderr


def build(verbose=False, force=False, ptxas_v=False):
    os.makedirs(OBJ, exist_ok=True)
    hdrs = [os.path.join(CSRC, f) for f in ("riccati_group.cuh", "riccati_launch.cuh", "riccati_configs.h",
                                            "vxx_layout.h")]
    hdrs.append(os.path.join(PKG, "..", "include", "aligator_b200", "gar.h"))
    hdrs_block = hdrs + [os.path.join(CSRC, f) for f in ("riccati_block.cuh", "riccati_block_launch.h",
                                                          "lq_assemble.h", "lq_adjoint.h", "lq_tangent.h", "lq_resolve.h",
                                                          "lq_resolve.cuh", "lq_factor_adjoint.h", "lq_factor_adjoint.cuh",
                                                          "lq_factor_tangent.h", "lq_factor_tangent.cuh",
                                                          "lq_jacobian.h", "lq_refine.h", "kkt_error.h",
                                                          "linesearch.h", "proxddp_inner.h")]
    extra = ["-Xptxas", "-v"] if ptxas_v else []
    jobs = []
    for (nx, nu, nc, g) in configs():
        src = os.path.join(CSRC, "kernel_inst.cu")
        tag = _digest(hdrs + [src], "%d_%d_%d_%d%s" % (nx, nu, nc, g, extra))
        obj = os.path.join(OBJ, "k_%d_%d_%d_%s.o" % (nx, nu, nc, tag))
        cmd = [NVCC] + ARCH + FLAGS + extra + ["-DAB2_NX=%d" % nx, "-DAB2_NU=%d" % nu, "-DAB2_NC=%d" % nc,
                                              "-DAB2_G=%d" % g, "-c", src, "-o", obj]
        jobs.append((obj, cmd))
    src = os.path.join(CSRC, "gar_cuda.cu")
    tag = _digest(hdrs_block + [src])
    obj = os.path.join(OBJ, "capi_%s.o" % tag)
    jobs.append((obj, [NVCC] + ARCH + FLAGS + ["-c", src, "-o", obj]))
    src = os.path.join(CSRC, "block_kernel.cu")
    obj = os.path.join(OBJ, "block_%s.o" % _digest(hdrs_block + [src], str(extra)))
    jobs.append((obj, [NVCC] + ARCH + FLAGS + extra + ["-c", src, "-o", obj]))
    src = os.path.join(CSRC, "kkt_error.cu")
    obj = os.path.join(OBJ, "kkt_%s.o" % _digest([os.path.join(CSRC, "kkt_error.h"), src], str(extra)))
    jobs.append((obj, [NVCC] + ARCH + FLAGS + extra + ["-c", src, "-o", obj]))
    src = os.path.join(CSRC, "lq_assemble.cu")
    obj = os.path.join(OBJ, "assemble_%s.o" % _digest([hdrs[-1], os.path.join(CSRC, "lq_assemble.h"), src], str(extra)))
    jobs.append((obj, [NVCC] + ARCH + FLAGS + extra + ["-c", src, "-o", obj]))
    src = os.path.join(CSRC, "lq_adjoint.cu")
    obj = os.path.join(OBJ, "adjoint_%s.o" % _digest([os.path.join(CSRC, "lq_adjoint.h"), src], str(extra)))
    jobs.append((obj, [NVCC] + ARCH + FLAGS + extra + ["-c", src, "-o", obj]))
    src = os.path.join(CSRC, "lq_tangent.cu")
    obj = os.path.join(OBJ, "tangent_%s.o" % _digest([os.path.join(CSRC, f) for f in ("lq_adjoint.h", "lq_tangent.h")]
                                                     + [src], str(extra)))
    jobs.append((obj, [NVCC] + ARCH + FLAGS + extra + ["-c", src, "-o", obj]))
    src = os.path.join(CSRC, "lq_resolve.cu")
    obj = os.path.join(OBJ, "resolve_%s.o" % _digest([os.path.join(CSRC, f) for f in ("vxx_layout.h", "lq_resolve.h",
                                                                                      "lq_resolve.cuh")]
                                                     + [src], str(extra)))
    jobs.append((obj, [NVCC] + ARCH + FLAGS + extra + ["-c", src, "-o", obj]))
    src = os.path.join(CSRC, "lq_factor_adjoint.cu")
    obj = os.path.join(OBJ, "factor_adjoint_%s.o" % _digest([os.path.join(CSRC, f) for f in (
        "vxx_layout.h", "lq_resolve.cuh", "item_launch.cuh", "lq_factor_adjoint.h", "lq_factor_adjoint.cuh")] + [src],
        str(extra)))
    jobs.append((obj, [NVCC] + ARCH + FLAGS + extra + ["-c", src, "-o", obj]))
    src = os.path.join(CSRC, "lq_factor_tangent.cu")
    obj = os.path.join(OBJ, "factor_tangent_%s.o" % _digest([os.path.join(CSRC, f) for f in (
        "vxx_layout.h", "lq_resolve.cuh", "item_launch.cuh", "lq_factor_tangent.h", "lq_factor_tangent.cuh")] + [src],
        str(extra)))
    jobs.append((obj, [NVCC] + ARCH + FLAGS + extra + ["-c", src, "-o", obj]))
    src = os.path.join(CSRC, "lq_jacobian.cu")
    obj = os.path.join(OBJ, "jacobian_%s.o" % _digest([os.path.join(CSRC, f) for f in ("lq_adjoint.h", "lq_jacobian.h",
                                                                                       "lq_record.cuh")]
                                                      + [src], str(extra)))
    jobs.append((obj, [NVCC] + ARCH + FLAGS + extra + ["-c", src, "-o", obj]))
    src = os.path.join(CSRC, "lq_refine.cu")
    obj = os.path.join(OBJ, "refine_%s.o" % _digest([os.path.join(CSRC, f) for f in ("lq_adjoint.h", "lq_refine.h",
                                                                                     "lq_record.cuh")]
                                                    + [src], str(extra)))
    jobs.append((obj, [NVCC] + ARCH + FLAGS + extra + ["-c", src, "-o", obj]))
    src = os.path.join(CSRC, "linesearch.cu")
    obj = os.path.join(OBJ, "linesearch_%s.o" % _digest([os.path.join(CSRC, "linesearch.h"), src], str(extra)))
    jobs.append((obj, [NVCC] + ARCH + FLAGS + extra + ["-c", src, "-o", obj]))
    src = os.path.join(CSRC, "proxddp_inner.cu")
    obj = os.path.join(OBJ, "inner_%s.o" % _digest([hdrs[-1], os.path.join(CSRC, "proxddp_inner.h"), src], str(extra)))
    jobs.append((obj, [NVCC] + ARCH + FLAGS + extra + ["-c", src, "-o", obj]))
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
