"""tests/test_workflow_timeout_gpu.py on the CPU emulator: the library compiled for tests/emu (same kernel and host
sources) behind the real C-ABI, in a child process, as tests/test_in_flight_emulator.py does for the hold in flight.
The 10 M-record comparison stays on the GPU."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402


def test_workflow_timeout_suite_on_the_emulated_library():
    got = emu_sweep.run_suite("tests/test_workflow_timeout_gpu.py", k="not full_size")
    assert got["passed"] >= 55, got


def test_timeout_call_sequences_on_the_emulated_library():
    got = emu_sweep.run_suite("tests/test_timeout_call_sequences_gpu.py", k="not full_size")
    assert got["passed"] >= 12, got


# world, idx_bytes, records in total, amgen config (22: named time zones, 3: remedy actions)
@pytest.mark.parametrize("case", [(2, 4, 20_000, 22), (3, 8, 30_011, 3)], ids=lambda c: "w{}_b{}_n{}_c{}".format(*c))
def test_each_shard_times_out_its_own_runs_through_am_gather_tick_view(case):
    """tests/emu/run_gather_timeout.py: every rank's global list against the timeout oracle of the unsharded population,
    and its am_sweep_last_timed_out the part it owns (every rank times out runs)"""
    emu_sweep.run_script("run_gather_timeout.py", case)
