"""Adversarial populations (tests/adversarial.py) for the sweep kernels on the CPU emulator (tests/emu)
against the oracle: counters and intervals at the i32 extremes, finishedAt on the due boundary, remedy
gates at the extremes, schedules bound to named time zones, T at 0, -1, 2^31, +-2^40, +-2^54 — and,
beyond what the library itself can produce, kinds 6/7, both PENDING bits at once, zero / negative
intervals and negative counters.  Three consecutive ticks, all four kernel variants (open/closed loop
x masks/no masks), bit-exact lists, statistics and columns.  The same cases run on the device in
tests/test_sweep_adversarial_gpu.py."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402
from adversarial import TS, ZoneMap, product_lookup, run_single_ticks  # noqa: E402


@pytest.fixture(scope="module")
def emu_zones():
    # zone ids of the emulated library's own registry
    return ZoneMap(product_lookup(emu_sweep.load()))


@pytest.mark.parametrize("in_domain", [True, False], ids=["library-domain", "beyond-domain"])
@pytest.mark.parametrize("seed", range(12))
def test_adversarial_population(emu_zones, seed, in_domain):
    for mode in (0, 1, 2, 3):  # closed loop / full scan bits
        bad = run_single_ticks(emu_sweep.EmuSweep, emu_zones, seed, 2500, TS[seed % len(TS)], mode, in_domain)
        assert bad is None, bad
