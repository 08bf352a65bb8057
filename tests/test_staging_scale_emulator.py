"""tests/test_staging_scale_gpu.py on the CPU emulator: the library compiled for tests/emu (same kernel and host
sources) behind the real C-ABI, in a child process."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402


def test_staging_scale_suite_on_the_emulated_library():
    got = emu_sweep.run_suite("tests/test_staging_scale_gpu.py")
    assert got["passed"] == 1, got
