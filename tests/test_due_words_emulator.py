"""tests/test_due_words_gpu.py on the CPU emulator: the library compiled for tests/emu (same kernel and host sources)
behind the real C-ABI, in a child process, on smaller handles for the walks (SEQ_CAPACITIES)."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402


def test_due_words_on_the_emulated_library():
    got = emu_sweep.run_suite("tests/test_due_words_gpu.py", env={"SEQ_CAPACITIES": "257,513,257,1025,129"})
    assert got["passed"] >= 9, got
