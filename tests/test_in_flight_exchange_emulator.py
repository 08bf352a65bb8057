"""Ticks with the hold in flight on, through the sharded whole step, am_gather_tick_view, on the CPU emulator's rank
threads (tests/emu/run_gather_hold.py, as tests/test_catch_up_exchange_emulator.py does for catch-up ticks): the hold
variants launched by am_sweep_tick_shard, their bitmap and exceptions through the exchange, every rank's global list
against the hold oracle of the unsharded population, and every rank's columns and in-flight slots afterwards."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402

# world, idx_bytes, records in total, amgen config (22: named time zones, 3: remedy actions, 2: the bench mix)
CASES = [(2, 4, 20_000, 22), (3, 8, 30_011, 3), (4, 4, 24_000, 2)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w{}_b{}_n{}_c{}".format(*c))
def test_sharded_ticks_with_the_hold_equal_the_hold_oracle_of_the_unsharded_population(case):
    emu_sweep.run_script("run_gather_hold.py", case)
