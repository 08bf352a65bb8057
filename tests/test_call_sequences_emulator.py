"""tests/test_call_sequences_gpu.py on the CPU emulator: the library compiled for tests/emu (same kernel and host
sources) behind the real C-ABI, in a child process, as tests/test_catch_up_emulator.py does for catch-up ticks.  The
walks run on smaller handles (SEQ_CAPACITIES); the emulated library completes every call before it returns, so the
walks tick on the handle's own stream only."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402


def test_call_sequences_on_the_emulated_library():
    got = emu_sweep.run_suite("tests/test_call_sequences_gpu.py", env={"SEQ_CAPACITIES": "1,257,1025,3001,513,2049"})
    assert got["passed"] >= 9, got
