"""Compiles and runs tests/cpp/test_reconciler.cpp — the C++ host-side mirror of the
reference's HealthCheckReconciler surface (include/amsweep_reconciler.hpp) — against
libamsweep.  The compile step also runs on CPU; running needs a GPU."""
import os
import subprocess

import pytest

from conftest import ROOT

SRC = os.path.join(ROOT, "tests", "cpp", "test_reconciler.cpp")
LIBDIR = os.path.join(ROOT, "active-monitor_b200", "lib")


def _build(tmp_path):
    """links the mirror into the test's temporary directory: the repository tree may be read-only"""
    exe = str(tmp_path / "test_reconciler.bin")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), SRC,
                    "-L", LIBDIR, "-lamsweep", f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


def test_reconciler_mirror_compiles(tmp_path):
    assert os.path.exists(_build(tmp_path))


@pytest.mark.gpu
def test_reconciler_mirror_behaves_like_the_reference_tests(tmp_path):
    exe = _build(tmp_path)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stdout + out.stderr
