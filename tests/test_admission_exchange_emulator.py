"""The submit budget through the sharded whole step, am_gather_tick_view, on the CPU emulator's rank threads
(tests/emu/run_gather_admission.py): each rank with its own budget and model; its global list, view, statistics, waits
and last admission against the models after every step.  The exchange must carry each shard's admitted list as it is."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402

# world, idx_bytes, records in total (30,011 over 3 ranks: shards cut inside groups and words), amgen config
CASES = [(2, 4, 20_000, 2), (3, 8, 30_011, 3)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w{}_b{}_n{}_c{}".format(*c))
def test_budgeted_shards_through_the_exchange_equal_their_models(case):
    emu_sweep.run_script("run_gather_admission.py", case)
