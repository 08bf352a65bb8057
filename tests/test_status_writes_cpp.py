"""Compiles and runs tests/cpp/test_status_writes.cpp — HealthCheckReconciler::StatusWrites of the C++ mirror
(include/amsweep_reconciler.hpp), the status writes built from the change details — against libamsweep.  The compile
step also runs on CPU; running needs a GPU."""
import os
import subprocess

import pytest

from conftest import ROOT

SRC = os.path.join(ROOT, "tests", "cpp", "test_status_writes.cpp")
LIBDIR = os.path.join(ROOT, "active-monitor_b200", "lib")


def _build(tmp_path):
    """links the mirror into the test's temporary directory: the repository tree may be read-only"""
    exe = str(tmp_path / "test_status_writes.bin")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), SRC,
                    "-L", LIBDIR, "-lamsweep", f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


def test_status_writes_compile(tmp_path):
    assert os.path.exists(_build(tmp_path))


@pytest.mark.gpu
def test_status_writes_follow_the_reference(tmp_path):
    exe = _build(tmp_path)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stdout + out.stderr
