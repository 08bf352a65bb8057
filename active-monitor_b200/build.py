"""In-tree build of the native pieces (no JIT cache, no pip install).

  active-monitor_b200/lib/libamsweep.so   product: CUDA sweep + C-ABI (nvcc, sm_90a)
  tools/amgen/libamgen.so                 neutral synthetic-population generator (gcc)
  oracle/_build/libamsweep_oracle.so      CPU oracle — test infrastructure (gcc)

The reference is Go (no toolchain in this image), so there is no oracle/_ref.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
LIB = os.path.join(LIBDIR, "libamsweep.so")
AMGEN = os.path.join(ROOT, "tools", "amgen", "libamgen.so")
ORACLE = os.path.join(ROOT, "oracle", "_build", "libamsweep_oracle.so")

SOURCES = ("sweep.cu", "gather.cu", "cron_parse.cpp", "handoff.cpp", "host_loops.cpp", "tz.cpp", "ingest_json.cpp")
HEADERS = ("sweep_kernels.cuh", "admission_kernels.cuh", "checkpoint_kernels.cuh", "checkpoint_pack_kernels.cuh", "sweep_block.cuh", "sweep_types.h", "sweep_internal.h", "gather_kernels.cuh", "civil.h", "tz.h", "tz_eval.h")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]


def _newer(target: str, sources: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _run(cmd: list[str], cwd: str | None = None) -> None:
    r = subprocess.run(cmd, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"build failed: {' '.join(cmd)}\n{r.stdout}")


def _nvcc() -> str:
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found: libamsweep cannot be built (there is no CPU fallback)")


def build_product(force: bool = False, verbose: bool = False) -> str:
    srcs = [os.path.join(CSRC, f) for f in SOURCES]
    deps = srcs + [os.path.join(CSRC, f) for f in HEADERS] + [
        os.path.join(ROOT, "include", "amsweep.h")]
    if force or _newer(LIB, deps):
        os.makedirs(LIBDIR, exist_ok=True)
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + srcs
        _run(cmd)
    return LIB


def build_amgen(force: bool = False) -> str:
    src = os.path.join(ROOT, "tools", "amgen", "amgen.c")
    if force or _newer(AMGEN, [src, os.path.join(ROOT, "include", "amsweep.h")]):
        _run(["gcc", "-O3", "-g", "-std=gnu11", "-Wall", "-fPIC", "-pthread", "-shared", "-o", AMGEN,
              src, "-lpthread"])
    return AMGEN


def build_oracle(force: bool = False) -> str:
    odir = os.path.join(ROOT, "oracle")
    if force or _newer(ORACLE, [os.path.join(odir, "amsweep_oracle.c"),
                                os.path.join(odir, "amsweep_oracle.h")]):
        _run(["make", "-C", odir, "-B"] if force else ["make", "-C", odir])
    return ORACLE


def build_all(force: bool = False, verbose: bool = False) -> dict:
    return {"libamsweep": build_product(force, verbose), "libamgen": build_amgen(force),
            "oracle": build_oracle(force)}


if __name__ == "__main__":
    out = build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    for k, v in out.items():
        print(f"{k}: {v}")
