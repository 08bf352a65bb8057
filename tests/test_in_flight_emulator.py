"""tests/test_in_flight_gpu.py on the CPU emulator: the library compiled for tests/emu (same kernel and host sources)
behind the real C-ABI, in a child process, as tests/test_catch_up_emulator.py does for catch-up ticks.  The 10 M-record
comparison stays on the GPU."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402


def test_in_flight_suite_on_the_emulated_library():
    got = emu_sweep.run_suite("tests/test_in_flight_gpu.py", k="not full_size")
    assert got["passed"] >= 30, got
