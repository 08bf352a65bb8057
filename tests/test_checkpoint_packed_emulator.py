"""tests/test_checkpoint_packed_gpu.py on the CPU emulator: the library compiled for tests/emu (same kernel and host
sources) behind the real C-ABI, in a child process, as tests/test_checkpoint_delta_emulator.py does."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402


def test_checkpoint_packed_suite_on_the_emulated_library():
    got = emu_sweep.run_suite("tests/test_checkpoint_packed_gpu.py", k="not full_size")
    assert got["passed"] >= 15, got
