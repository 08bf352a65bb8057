"""tests/test_select_gpu.py on the CPU emulator: the library compiled for tests/emu (same kernel and host sources) behind
the real C-ABI, in a child process.  The 10 M-record comparison and the tick on a caller stream stay on the GPU."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402


def test_select_suite_on_the_emulated_library():
    got = emu_sweep.run_suite("tests/test_select_gpu.py", k="not full_size and not caller_stream")
    assert got["passed"] >= 9, got
