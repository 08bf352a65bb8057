"""Catch-up ticks (AM_SWEEP_CATCH_UP) through the sharded whole step, am_gather_tick_view, on the CPU emulator's rank
threads (tests/emu/run_gather_catch_up.py, as tests/test_exchange_emulator.py does for plain ticks): the window
variant launched by am_sweep_tick_shard, its bitmap, exceptions and statistics through the exchange, every rank's
global list against the window oracle of the unsharded population, and every rank's P afterwards."""
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


# world, idx_bytes, records in total, amgen config (22: named time zones, 3: remedy actions), closed loop
CASES = [(2, 4, 20_000, 22, 0), (3, 8, 30_011, 22, 1), (4, 4, 24_000, 3, 0), (2, 8, 16_000, 3, 1)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w{}_b{}_n{}_c{}_closed{}".format(*c))
def test_sharded_catch_up_ticks_equal_the_window_oracle_of_the_unsharded_population(emu_lib, case):
    out = subprocess.run([sys.executable, os.path.join(EMU, "run_gather_catch_up.py")] + [str(a) for a in case],
                         cwd=ROOT, env=dict(os.environ, AMSWEEP_LIB=emu_lib), capture_output=True, text=True,
                         timeout=900)
    assert out.returncode == 0 and out.stdout.strip().startswith("ok"), out.stdout[-3000:] + out.stderr[-3000:]
