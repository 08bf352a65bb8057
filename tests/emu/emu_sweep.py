"""The WHOLE product library on the CPU emulator, in-process: csrc/*.cu + kernels compiled against
tests/emu/cuda_emu.h (execution model) and tests/emu/cuda_rt_emu.h (runtime calls) into
tests/emu/libamsweep_emu.so, and `EmuSweep` = `am.Sweep` bound to that library instead of the CUDA
build — same C-ABI, same host runtime, same kernel source.  Test infrastructure only.

(Round 1 kept a second, kernel-only harness here that restated the launch sequence of sweep.cu;
it is gone: the real launch sequence runs on the emulator.)"""
import ctypes as C
import importlib
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "active-monitor_b200", "csrc")
LIB = os.path.join(HERE, "libamsweep_emu.so")
_lib = None


def sources():
    b = importlib.import_module("active-monitor_b200.build")
    return [os.path.join(CSRC, f) for f in b.SOURCES], [os.path.join(CSRC, f) for f in b.HEADERS]


def build():
    srcs, hdrs = sources()
    deps = srcs + hdrs + [os.path.join(HERE, "cuda_emu.h"), os.path.join(HERE, "cuda_rt_emu.h"),
                          os.path.join(ROOT, "include", "amsweep.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wno-unknown-pragmas", "-pthread", "-fPIC", "-shared",
                        # same-named symbols exist in libamsweep.so (loaded RTLD_GLOBAL by the tests): bind locally
                        "-Wl,-Bsymbolic",
                        "-DAMSWEEP_EMULATE", "-include", os.path.join(HERE, "cuda_emu.h"),
                        "-include", os.path.join(HERE, "cuda_rt_emu.h"), "-x", "c++"] + srcs + ["-o", LIB],
                       check=True)
    return LIB


def build_tsan(main_cpp, out):
    """tests/emu/<main_cpp> with the library's own sources on the emulator, built with -fsanitize=thread into `out`
    (the emulator tells TSan about its fibers); skips the test when the toolchain has no ThreadSanitizer runtime"""
    import pytest
    srcs = sources()[0] + [os.path.join(HERE, main_cpp)]
    r = subprocess.run(["g++", "-std=c++20", "-O1", "-g", "-fsanitize=thread", "-Wno-unknown-pragmas", "-Wno-tsan",
                        "-pthread", "-DAMSWEEP_EMULATE", "-include", os.path.join(HERE, "cuda_emu.h"),
                        "-include", os.path.join(HERE, "cuda_rt_emu.h"), "-x", "c++"] + srcs + ["-o", out],
                       capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("ThreadSanitizer runtime not available: " + r.stderr[-300:])
    return out


def _child(cmd, env, timeout):
    return subprocess.run([sys.executable] + cmd, cwd=ROOT, env=dict(os.environ, AMSWEEP_LIB=build(), **(env or {})),
                          capture_output=True, text=True, timeout=timeout)


def run_script(name, args, env=None, timeout=900):
    """tests/emu/<name> with `args` on the emulated library, in a child process: it must exit 0 and print "ok ..."
    first; returns its stdout"""
    out = _child([os.path.join(HERE, name)] + [str(a) for a in args], env, timeout)
    assert out.returncode == 0 and out.stdout.strip().startswith("ok"), out.stdout[-3000:] + out.stderr[-3000:]
    return out.stdout


def run_suite(paths, k=None, env=None, timeout=1800, allow=()):
    """the `-m gpu` tests of `paths` on the emulated library, in a child pytest that must pass.  Returns its summary
    line as counts, e.g. {"passed": 61, "deselected": 2}; an outcome other than passed that is not in `allow`
    (failed, error, skipped, xfailed, ...) fails the call."""
    out = _child(["-m", "pytest"] + ([paths] if isinstance(paths, str) else list(paths)) +
                 ["-m", "gpu", "-q", "-x", "-p", "no:cacheprovider"] + (["-k", k] if k else []), env, timeout)
    tail = out.stdout[-3000:] + out.stderr[-2000:]
    assert out.returncode == 0, tail
    counts = {}
    for part in out.stdout.strip().splitlines()[-1].strip("= ").split(" in ")[0].split(", "):
        n, what = part.split()
        counts[what.rstrip("s") if what in ("errors", "warnings") else what] = int(n)
    assert counts.get("passed", 0) > 0 and set(counts) <= {"passed", "deselected", "warning", *allow}, tail
    return counts


def load():
    global _lib
    if _lib is None:
        abi = importlib.import_module("active-monitor_b200._lib")
        lib = C.CDLL(build(), mode=os.RTLD_LOCAL)
        for name, (res, args) in abi.SYMBOLS.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        # this second copy of the library has its own time-zone registry: introduce the generator's
        # zones in the generator's order, so that records classified by the CUDA build of the
        # library (the tests do that) carry ids this copy understands
        sys.path.insert(0, os.path.join(ROOT, "tools", "amgen"))
        import amgen
        for z in amgen.ZONES:
            i = C.c_int32()
            assert lib.am_tz_lookup(z.encode(), len(z), C.byref(i)) == 0
        _lib = lib
    return _lib


def _sweep_class():
    am = importlib.import_module("active-monitor_b200")

    class EmuSweep(am.Sweep):
        def __init__(self, capacity: int, shard_base: int = 0):
            super().__init__(capacity, device=0, shard_base=shard_base, lib=load())

        def tick(self, unix_sec, mode=0, cap=None, buffers=None):
            """like am.Sweep.tick, but a short buffer returns the partial list (the kernel-level
            harness of round 1 did) instead of raising"""
            try:
                return super().tick(unix_sec, mode, cap, buffers)
            except am.AmError as e:
                if e.code != am.AM_E_NOSPACE:
                    raise
                return e.partial

    return EmuSweep


def EmuSweep(capacity: int, shard_base: int = 0):
    return _sweep_class()(capacity, shard_base)
