"""Compare the generated code of two builds of the library, kernel by kernel.

    python tools/compare_sass.py OLD_BUILD_DIR NEW_BUILD_DIR

The arguments are two `aligator_b200/csrc/build` directories.  Objects are matched by name without their digest
(`k_12_6_0_<digest>.o` -> `k_12_6_0`).  Each object is disassembled with `cuobjdump -sass`; addresses and file
names are dropped, so a change of line tables alone (the build uses -lineinfo) compares equal, while every
instruction and its encoding (which carries the scheduling control bits) must match.  Prints one JSON line: per
object, the kernels that differ or exist on one side only.  Exits 1 when a sweep object (the per-shape `k_*`
objects and `block`, which holds the CTA-per-instance, static, parametric, leg and dense kernels) differs; the other
objects are reported only."""
import glob
import json
import os
import re
import subprocess
import sys

CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
SWEEPS = re.compile(r"^(k_\d+_\d+_\d+|block)$")


def objects(build):
    return {re.sub(r"_[0-9a-f]{16}$", "", os.path.basename(p)[:-2]): p for p in glob.glob(os.path.join(build, "*.o"))}


def kernels(obj):
    """{function name: [normalised SASS lines]}"""
    out = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    res, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = res.setdefault(m.group(1), [])
            continue
        if cur is None or "identifier" in line:
            continue
        line = re.sub(r"/\*[0-9a-f]{4,}\*/", "", line).strip()  # instruction address
        if line:
            cur.append(line)
    return res


def main():
    old, new = objects(sys.argv[1]), objects(sys.argv[2])
    report, fail, same = {}, False, 0
    for name in sorted(set(old) | set(new)):
        if name not in old or name not in new:
            report[name] = "only in %s" % ("old" if name in old else "new")
            fail |= bool(SWEEPS.match(name))
            continue
        a, b = kernels(old[name]), kernels(new[name])
        diff = sorted(k for k in set(a) | set(b) if a.get(k) != b.get(k))
        same += len(set(a) & set(b)) - len([k for k in diff if k in a and k in b])
        if diff:
            report[name] = diff
            fail |= bool(SWEEPS.match(name))
    print(json.dumps(dict(identical_kernels=same, differing=report, sweeps_identical=not fail)))
    return 1 if fail else 0


if __name__ == "__main__":
    sys.exit(main())
