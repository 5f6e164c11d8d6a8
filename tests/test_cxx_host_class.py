"""The C++ host class (include/aligator_b200/riccati_solver.hpp): compiles and links
against the C-ABI library on CPU; runs its parity checks on the GPU box."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cxx", "host_class_test.cpp")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    """The test program, built outside the source tree (which may be read-only)."""
    import __graft_entry__ as g
    g.build()
    libdir = os.path.join(ROOT, "aligator_b200")
    path = str(tmp_path_factory.mktemp("cxx") / "host_class_test")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-Wall", SRC, "-o", path,
                           "-L" + libdir, "-laligator_b200_gar", "-Wl,-rpath," + libdir])
    return path


def test_host_class_compiles_and_links(exe):
    assert os.path.exists(exe)


@pytest.mark.gpu
def test_host_class_parity_on_gpu(exe):
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ALL OK" in r.stdout
