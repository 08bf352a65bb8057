"""The whole product library — csrc/sweep.cu (handle, staging, drain, tick, read, run_ticks, ...)
with csrc/sweep_kernels.cuh, and csrc/gather.cu with gather_kernels.cuh — compiled for the CPU emulator (tests/emu/cuda_emu.h for the kernels,
tests/emu/cuda_rt_emu.h for the dozen CUDA runtime calls) into tests/emu/libamsweep_emu.so, and the
GPU parity tests run against it THROUGH THE REAL C-ABI in a child process (AMSWEEP_LIB points the
ctypes layer at it).  Same sources as the shipped library: only the kernel-launch macro and three
inline-PTX helpers differ (#ifdef AMSWEEP_EMULATE), and the shipped build is byte-identical with
and without those guards.

So `-m "not gpu"` now exercises the host runtime and the kernels' logic end to end; the `-m gpu`
run on an H100 remains the parity test proper (memory model, real launches, real streams).
Skipped here: the torch.cuda-based tick_device test, the two 10 M-record compares (a minute of emulation for
no logic the smaller sizes do not reach; they run on the GPU) and the stream tests of test_device_pipeline_gpu.py
(the emulator completes every call before it returns; its misalignment test runs here).
"""
import os
import subprocess
import sys

import pytest

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import emu_sweep  # noqa: E402

EMU = emu_sweep.HERE


@pytest.fixture(scope="module")
def emu_lib():
    return emu_sweep.build()


def test_emulated_library_exports_the_whole_abi(emu_lib):
    import ctypes as C
    import importlib
    abi = importlib.import_module("active-monitor_b200._lib")
    lib = C.CDLL(emu_lib, mode=os.RTLD_LOCAL)
    for name in abi.SYMBOLS:
        assert hasattr(lib, name), name


def test_gpu_parity_suite_through_the_c_abi_on_the_emulated_library():
    got = emu_sweep.run_suite(["tests/test_sweep_gpu.py", "tests/test_golden_fixtures.py", "tests/test_timezones.py",
                               "tests/test_sweep_adversarial_gpu.py", "tests/test_device_pipeline_gpu.py"],
                              k="not tick_device and not 10m", allow=("skipped",))
    assert got["passed"] >= 135, got


def test_reconciler_cpp_mirror_on_the_emulated_library(emu_lib):
    """tests/cpp/test_reconciler.cpp (the C++ mirror of the reference's reconciler tests) linked
    against the emulated library."""
    exe = os.path.join(ROOT, "tests", "cpp", "test_reconciler_emu.bin")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "test_reconciler.cpp"), "-L", EMU, "-lamsweep_emu",
                    f"-Wl,-rpath,{EMU}", "-pthread", "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stdout + out.stderr


def test_random_call_sequences_against_a_sequential_model():
    """tests/emu/fuzz_c_abi.py: random upsert / remove / post_result / read / tick sequences (duplicate
    slots, results before and after upserts, removes of absent slots, short output buffers, open and
    closed loop, a shard base) through am.Sweep on the emulated library; every tick and every read must
    equal the sequential model (calls take effect in call order; a tick is the oracle's sweep)."""
    emu_sweep.run_script("fuzz_c_abi.py", [60, 30, 3000])


def test_threading_contract_under_threadsanitizer(tmp_path):
    """tests/emu/tsan_c_abi.cpp: four threads stage upserts / removes / results while one thread ticks
    and reads (the contract of SURVEY 8b), built with -fsanitize=thread from the library's own sources
    on the emulator.  No ThreadSanitizer report = the host runtime's locking covers every shared access."""
    exe = emu_sweep.build_tsan("tsan_c_abi.cpp", str(tmp_path / "tsan_c_abi.bin"))
    out = subprocess.run([exe], capture_output=True, text=True, timeout=900,
                         env=dict(os.environ, TSAN_OPTIONS="halt_on_error=0"))
    assert "ThreadSanitizer" not in out.stderr, out.stderr[-3000:]
    assert out.returncode == 0 and out.stdout.startswith("ok"), out.stdout + out.stderr[-2000:]
