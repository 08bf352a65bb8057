"""Ticks with the hold in flight on, through the sharded whole step, am_gather_tick_view, on the CPU emulator's rank
threads (tests/emu/run_gather_hold.py, as tests/test_catch_up_exchange_emulator.py does for catch-up ticks): the hold
variants launched by am_sweep_tick_shard, their bitmap and exceptions through the exchange, every rank's global list
against the hold oracle of the unsharded population, and every rank's columns and in-flight slots afterwards."""
import os
import subprocess
import sys

import pytest

from conftest import ROOT

EMU = os.path.join(ROOT, "tests", "emu")


@pytest.fixture(scope="module")
def emu_lib():
    sys.path.insert(0, EMU)
    import emu_sweep
    return emu_sweep.build()


# world, idx_bytes, records in total, amgen config (22: named time zones, 3: remedy actions, 2: the bench mix)
CASES = [(2, 4, 20_000, 22), (3, 8, 30_011, 3), (4, 4, 24_000, 2)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w{}_b{}_n{}_c{}".format(*c))
def test_sharded_ticks_with_the_hold_equal_the_hold_oracle_of_the_unsharded_population(emu_lib, case):
    out = subprocess.run([sys.executable, os.path.join(EMU, "run_gather_hold.py")] + [str(a) for a in case],
                         cwd=ROOT, env=dict(os.environ, AMSWEEP_LIB=emu_lib), capture_output=True, text=True,
                         timeout=900)
    assert out.returncode == 0 and out.stdout.strip().startswith("ok"), out.stdout[-3000:] + out.stderr[-3000:]
