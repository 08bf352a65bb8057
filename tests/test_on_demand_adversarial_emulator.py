"""tests/test_on_demand_adversarial_gpu.py on the CPU emulator: the library compiled for tests/emu (same kernel and host
sources) behind the real C-ABI, in a child process, as tests/test_workflow_timeout_emulator.py does for the workflow
timeouts.  The 10 M-record next_due case stays on the GPU."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402


def test_on_demand_adversarial_suite_on_the_emulated_library():
    got = emu_sweep.run_suite("tests/test_on_demand_adversarial_gpu.py", k="not 10m", allow=("xfailed",))
    assert got["xfailed"] == 1, got  # the half-hour daylight-saving gap
    assert got["passed"] >= 249, got
