"""Compiles and runs tests/cpp/test_reconciler_spec.cpp — the spec path of the C++ mirror of the reconciler
(include/amsweep_reconciler.hpp, ProcessSpec) — against libamsweep on a GPU, and against the emulated library."""
import os
import subprocess
import sys

import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import emu_sweep  # noqa: E402

SRC = os.path.join(ROOT, "tests", "cpp", "test_reconciler_spec.cpp")


def _build(tmp_path, libdir, lib, extra=()):
    """links the test into the test's temporary directory: the repository tree may be read-only"""
    exe = str(tmp_path / "test_reconciler_spec.bin")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), SRC,
                    "-L", libdir, f"-l{lib}", f"-Wl,-rpath,{libdir}", *extra, "-o", exe], check=True)
    return exe


def _run(exe):
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stdout + out.stderr


def test_spec_path_on_the_emulated_library(tmp_path):
    lib = emu_sweep.build()
    _run(_build(tmp_path, os.path.dirname(lib), "amsweep_emu", ("-pthread",)))


@pytest.mark.gpu
def test_spec_path_keeps_a_posted_result(tmp_path):
    _run(_build(tmp_path, os.path.join(ROOT, "active-monitor_b200", "lib"), "amsweep"))
