"""Catch-up ticks (AM_SWEEP_CATCH_UP) through the sharded whole step, am_gather_tick_view, on the CPU emulator's rank
threads (tests/emu/run_gather_catch_up.py, as tests/test_exchange_emulator.py does for plain ticks): the window
variant launched by am_sweep_tick_shard, its bitmap, exceptions and statistics through the exchange, every rank's
global list against the window oracle of the unsharded population, and every rank's P afterwards."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402

# world, idx_bytes, records in total, amgen config (22: named time zones, 3: remedy actions), closed loop
CASES = [(2, 4, 20_000, 22, 0), (3, 8, 30_011, 22, 1), (4, 4, 24_000, 3, 0), (2, 8, 16_000, 3, 1)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w{}_b{}_n{}_c{}_closed{}".format(*c))
def test_sharded_catch_up_ticks_equal_the_window_oracle_of_the_unsharded_population(case):
    emu_sweep.run_script("run_gather_catch_up.py", case)
