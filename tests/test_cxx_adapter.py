"""The reference-side adapter (integration/aligator/gar/b200-riccati.hpp -- what a maintainer adds to aligator)
compiled against stand-in Eigen / aligator types (tests/cxx/aligator_stub; the image has no Eigen): compiles and
links against the C-ABI library on CPU, runs its parity checks against the oracle on the GPU box."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cxx", "adapter_test.cpp")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    """The test program, built outside the source tree (which may be read-only)."""
    import __graft_entry__ as g
    g.build()
    libdir = os.path.join(ROOT, "aligator_b200")
    path = str(tmp_path_factory.mktemp("cxx") / "adapter_test")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-Wall", SRC, "-o", path,
                           "-I" + os.path.join(ROOT, "tests", "cxx", "aligator_stub"), "-I" + os.path.join(ROOT, "integration"),
                           "-I" + os.path.join(ROOT, "include"),
                           "-L" + libdir, "-laligator_b200_gar", "-Wl,-rpath," + libdir])
    return path


def test_adapter_compiles_and_links(exe):
    assert os.path.exists(exe)


@pytest.mark.gpu
def test_adapter_parity_on_gpu(exe):
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ADAPTER OK" in r.stdout
