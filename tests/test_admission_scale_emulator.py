"""tests/test_admission_scale_gpu.py on the CPU emulator: the library compiled for tests/emu (same kernel and host
sources) behind the real C-ABI, in a child process.  The GPU-only cases (full_size, and the one-GPU world of the exchange, which needs torch on a device) stay on the GPU."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402


def test_admission_scale_suite_on_the_emulated_library():
    got = emu_sweep.run_suite("tests/test_admission_scale_gpu.py", k="not full_size and not one_gpu_world")
    assert got["passed"] == 13, got
