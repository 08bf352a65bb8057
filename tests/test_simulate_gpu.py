"""am_sweep_simulate against its oracle (tests/sim_driver.py, the contract's loop of posts and ticks on the handle model),
tick by tick and blocked: every statistics row and simulated row, all sixteen columns, am_sweep_in_flight and
am_sweep_remedy_in_flight after the call, then plain ticks that go on from where the simulation left the runs (the pair
compares everything after each, the timed-out lists included).  On the adversarial population with remedies, limits,
reset intervals and workflow timeouts, durations of 1-5 s so that ends meet deadlines, cron minutes and each other, runs
started by real ticks before the call (some overdue at its first tick), results staged before it, several block
lengths, a daylight-saving transition, every refusal, and 10 M records."""
import os
import sys

import numpy as np
import pytest

import sim_driver
from adversarial import ZoneMap, population, zones_usable
from handle_model import Refused
from handle_pair import Pair, emulated

pytestmark = pytest.mark.gpu

DAY = 86400
T_OCT = 1790812800 + 37  # 2026-10-01 00:00:37 UTC
T_DST = 1792371600 - 90  # 90 s before 2026-10-25 01:00 UTC (Europe leaves summer time)
BLOCKED = sim_driver.BLOCKED
SHORT = (1, 5, 1, 4)


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def _records(am, rng, n, T, zmap):
    recs = am.columns_to_records(population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))))
    # timeouts on some, remedies with limits and reset intervals come with the population; some records get both
    recs["wf_timeout"] = np.where(rng.random(n) < 0.5, 0, rng.integers(1, 6, n))
    return recs


def _compare(am, p, got, want, what):
    (rows, sims), (wrows, wsims) = got, want
    assert len(rows) == len(wrows)
    for k, (r, w) in enumerate(zip(rows, wrows)):
        gd = {f: int(r[f]) for f in am.abi.STAT_FIELDS}
        assert gd == w, (what, k, {f: (gd[f], w[f]) for f in gd if gd[f] != w[f]})
    np.testing.assert_array_equal(np.array([tuple(s) for s in sims], dtype=np.int64).reshape(-1, 4),
                                  np.array(wsims, dtype=np.int64).reshape(-1, 4), err_msg=f"{what}: sim rows")
    dev = p.s.read_range(0, p.n)
    for name in am.COLUMN_NAMES:
        np.testing.assert_array_equal(dev[name], p.m.cols()[name], err_msg=f"{what}: {name}")
    np.testing.assert_array_equal(p.s.in_flight(0, p.n), p.m.in_flight(0, p.n), err_msg=f"{what}: in flight")
    np.testing.assert_array_equal(p.s.remedy_in_flight(0, p.n), p.m.remedy_in_flight(0, p.n),
                                  err_msg=f"{what}: remedy in flight")
    for k in range(2):
        assert len(p.s.last_timed_out()[k]) == 0 and len(p.s.last_remedy_timed_out()[k]) == 0


def _both(am, p, T0, n, mode, seed, params):
    want = sim_driver.simulate(p.m, T0, n, mode, seed, params)
    got = p.s.simulate(T0, n, mode, seed, params)
    _compare(am, p, got, want, (mode, T0, n))
    return got


def _setup(am, zmap, rng, n, T0, started=True):
    """a handle with both holds, the population upserted, runs started by real ticks before T0 (with durations of at
    most 5 s the ones from T0 - 6 are overdue at T0) and results staged before the call"""
    p = Pair(am, zmap, n, hold=True, remedy=True)
    p.upsert(np.arange(n), _records(am, rng, n, T0, zmap))
    if started:
        for T in (T0 - 6, T0 - 2):
            p.tick(T)
    sl = rng.choice(n, n // 10, replace=False)
    p.post(sl, rng.integers(0, 3, len(sl)).astype(np.uint8), rng.integers(0, 3, len(sl)).astype(np.uint8))
    return p


def _go_on(am, p, T, ticks=70):
    """plain ticks after the simulation: the pair compares list, statistics, columns, both in-flight answers and both
    timed-out lists; next_due never lies past the first tick that does anything"""
    first = p.m.first_active_tick(T - 1, 120)
    nd = p.s.next_due(T - 1)
    assert first is None or nd <= first, (nd, first)
    timed = 0
    for t in range(T, T + ticks):
        p.tick(t)
        timed += len(p.m.last.timed_out[0]) + len(p.m.last.remedy_timed_out[0])
    return timed


@pytest.mark.parametrize("mode,block", [(0, 96), (BLOCKED, 1), (BLOCKED, 7), (BLOCKED, 96), (BLOCKED, 128)],
                         ids=["ticks", "blocked-1", "blocked-7", "blocked-96", "blocked-128"])
def test_adversarial_against_the_driver(am, zmap, monkeypatch, mode, block):
    monkeypatch.setenv("AMSWEEP_BLOCK_TICKS", str(block))
    rng = np.random.default_rng(block * 7 + mode)
    n = 640
    p = _setup(am, zmap, rng, n, T_OCT)
    try:
        _, sims = _both(am, p, T_OCT, 251, mode, 5 + block, SHORT)  # (not a multiple of any block length)
        sims = np.array([tuple(s) for s in sims])
        assert sims[:, 0].max() > 0 and sims[:, 1].max() > 0 and sims[:, 2].sum() > 0 and sims[:, 3].sum() > 0, sims.sum(0)
        # a second call on the same handle continues the runs, then plain ticks time out what it started
        _both(am, p, T_OCT + 251, 40, mode | 0x2, 11, (2, 9, 3, 12))
        _go_on(am, p, T_OCT + 291)
    finally:
        p.close()


@pytest.mark.parametrize("mode", [0, BLOCKED], ids=["ticks", "blocked"])
def test_daylight_saving_transition(am, zmap, mode):
    rng = np.random.default_rng(31 + mode)
    p = _setup(am, zmap, rng, 384, T_DST)
    try:
        _both(am, p, T_DST, 200, mode, 3, SHORT)
        _go_on(am, p, T_DST + 200, 30)
    finally:
        p.close()


@pytest.mark.parametrize("mode", [0, BLOCKED], ids=["ticks", "blocked"])
def test_long_runs_across_blocks(am, zmap, mode):
    """durations longer than a block: runs held for whole blocks, deadlines far ahead, nothing started before"""
    rng = np.random.default_rng(77 + mode)
    p = _setup(am, zmap, rng, 512, T_OCT, started=False)
    try:
        _both(am, p, T_OCT, 400, mode, 9, (90, 200, 50, 300))
        _go_on(am, p, T_OCT + 400, 20)
    finally:
        p.close()


REFUSALS = [
    ("hold off", dict(hold=False), 0, (1, 1, 1, 1), T_OCT),
    ("remedy hold off", dict(remedy=False), 0, (1, 1, 1, 1), T_OCT),
    ("wf_min 0", {}, 0, (0, 1, 1, 1), T_OCT),
    ("wf_max < wf_min", {}, 0, (3, 2, 1, 1), T_OCT),
    ("remedy_min 0", {}, 0, (1, 1, 0, 1), T_OCT),
    ("remedy_max < remedy_min", {}, 0, (1, 1, 5, 4), T_OCT),
    ("no params", {}, 0, None, T_OCT),
    ("closed loop", {}, 0x1, (1, 1, 1, 1), T_OCT),
    ("catch up", {}, 0x8, (1, 1, 1, 1), T_OCT),
    ("unknown bit", {}, 0x10, (1, 1, 1, 1), T_OCT),
    ("range", {}, 0, (1, 1, 1, 1), 1 << 55),
]


@pytest.mark.parametrize("case", REFUSALS, ids=[c[0] for c in REFUSALS])
def test_refusals_change_nothing(am, zmap, case):
    _, switches, mode, params, T0 = case
    rng = np.random.default_rng(3)
    p = _setup(am, zmap, rng, 256, T_OCT)
    try:
        if switches.get("remedy") is False:
            p.set_remedy(False)
        if switches.get("hold") is False:
            p.set_hold(False)
        with pytest.raises(Refused) as want:
            sim_driver.simulate(p.m, T0, 10, mode, 1, params)
        with pytest.raises(am.AmError) as got:
            if params is None:
                lib = p.s._lib
                st = np.zeros(10, dtype=am.abi.STATS_DTYPE)
                rc = lib.am_sweep_simulate(p.s._h, T0, 10, mode, 1, None, st.ctypes.data, None)
                p.s._check(rc, "am_sweep_simulate")
            else:
                p.s.simulate(T0, 10, mode, 1, params)
        assert got.value.code == want.value.code
        # nothing drained, P unchanged: the staged results and the runs are still there for the next tick
        p.tick(T_OCT + 1)
    finally:
        p.close()


def test_full_size(am):
    """10 M config-5 records with a seeded tenth given workflow timeouts: a simulated hour, blocked and tick by tick,
    bit-exact on statistics, simulated rows, columns and both in-flight answers"""
    if emulated(am):
        pytest.skip("10 M records: GPU only")
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import run_sim
    got = run_sim.compare(am, n=10_000_000, seconds=3600, seed=1)
    assert got["equal"], got
    assert got["peak_in_flight"] > 0 and got["timed_out"] > 0, got
