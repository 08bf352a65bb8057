"""Workflow timeouts (am_record_t.wf_timeout with the hold in flight on): a held run that outlives its deadline is
treated at the first tick past it as if Failed had been posted.  Compared after every tick with the model
(tests/handle_model.py, tests/handle_pair.py) — list, statistics, all sixteen columns, am_sweep_in_flight and am_sweep_last_timed_out —
through every tick entry point: the hand-derived cases, long random sequences on the adversarial population, next_due
against brute force, the refusals, the hold off, launch counts, and 10 M records."""
import zlib

import numpy as np
import pytest

import amgen
import timeout_cases
from adversarial import ZoneMap, population, zones_usable
from handle_pair import Pair, emulated

pytestmark = pytest.mark.gpu

DAY, HOUR = 86400, 3600
T_OCT = 1790812800  # 2026-10-01 00:00:00 UTC
NONE = timeout_cases.NONE
FULL, CATCH = 0x2, 0x8
ENTRIES = ["tick", "tick_view", "tick_device", "tick_shard"]


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def _empty(am, n):
    cols = am.records_to_columns(np.zeros(n, dtype=am.RECORD_DTYPE))
    cols["flags"][:] = am.F_TOMBSTONE
    return cols


# ---- 1. the hand-derived cases, through every tick entry point ------------------------------------------------------
@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("case", timeout_cases.CASES, ids=lambda c: c.__name__)
def test_hand_derived_cases(am, zmap, case, entry):
    p = Pair(am, zmap, _empty(am, 8), hold=True, entry=entry)
    try:
        case(am, p)
    finally:
        p.close()


# ---- 2. long random sequences on the adversarial population ---------------------------------------------------------
STEPS = [1, 1, 1, 57, 1, 1, 60, 2, 1, -60, 0, 1, 17, 1, 1, 59, 1, 0, 1, 600, 1, 1, 43, 1, -1, 1, 120, 1, 1, 30, 1, 29, 1,
         3600 + 17, 1, 1, 5, 55, 1]


def _records(am, rng, n, T, zmap, wmax):
    recs = am.columns_to_records(population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))))
    recs["wf_timeout"] = np.where(rng.random(n) < 0.2, 0, rng.integers(1, wmax, n))
    return recs


@pytest.mark.parametrize("mode", [0, FULL, CATCH, CATCH | FULL], ids=["plain", "full_scan", "catch_up", "catch_up_full"])
@pytest.mark.parametrize("entry", ENTRIES + ["short_buffer"])
def test_random_sequences_equal_the_oracle(am, zmap, entry, mode):
    n = 3000
    rng = np.random.default_rng(zlib.crc32(f"timeout {entry} {mode}".encode()))
    T = T_OCT + 12 * DAY + 14 * HOUR - 3
    cols = population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY)))
    p = Pair(am, zmap, cols, hold=True, entry="tick_short" if entry == "short_buffer" else entry, cap=5)
    try:
        # W on most records from the start (a load sets none: upsert them)
        sl = np.arange(n)
        p.upsert(sl, _records(am, rng, n, T, zmap, 120))
        for k, step in enumerate(STEPS):
            if k:
                r = rng.random()
                if r < 0.3:
                    sl = rng.choice(n, 60, replace=False)
                    p.upsert(sl, _records(am, rng, 60, T, zmap, 200))
                elif r < 0.4:
                    p.remove(rng.choice(n, 30, replace=False))
                elif r < 0.5:
                    first = int(rng.integers(0, n - 200))
                    p.load(first, population(rng, 200, T, True, zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))))
                elif r < 0.53:
                    p.set_hold(False)
                    p.set_hold(True)
                fl = np.flatnonzero(p.m.since != NONE)
                if len(fl) and k % 2:
                    dense = k % 5 == 3
                    sl = rng.choice(fl, min(len(fl), 2000 if dense else 30), replace=False)
                    if dense:  # over an eighth of the records: applied inside the sweep
                        sl = np.concatenate([sl, rng.choice(n, 500, replace=False)])
                    p.post(sl, rng.integers(0, 3, len(sl)).astype(np.uint8), rng.integers(0, 3, len(sl)).astype(np.uint8))
            T += step
            p.tick(T, mode)
        assert p.timed_total > 100, p.timed_total
    finally:
        p.close()


# ---- 3. next_due counts expiries as events ---------------------------------------------------------------------------
def test_next_due_counts_expiries(am, zmap):
    T = T_OCT + 10 * HOUR + 20
    rec = timeout_cases.rec
    recs = np.concatenate([rec(am, 45, repeat_after_sec=600, finished_at=T - 1000),
                           rec(am, 7, repeat_after_sec=3600, finished_at=T - 5000),
                           rec(am, 0, repeat_after_sec=300, finished_at=T - 1000),
                           rec(am, 200, cron="*/5 * * * *"),
                           rec(am, 90, cron="7 * * * *")])
    p = Pair(am, zmap, _empty(am, len(recs)), hold=True)
    try:
        p.upsert(np.arange(len(recs)), recs)
        checked = 0
        for step, post in [(0, None), (1, None), (3, [2]), (5, None), (30, None), (1, None), (200, [0])]:
            T += step
            if post:
                p.post(post, [am.PHASE_SUCCEEDED] * len(post))
            p.tick(T)
            nd = p.s.next_due(T)
            want = p.m.first_active_tick(T, 4000)
            assert nd == want, (T, nd, want)
            checked += 1
        assert checked == 7
    finally:
        p.close()


# ---- 4. refusals, the hold off, launch counts --------------------------------------------------------------------------
def test_a_negative_timeout_is_refused_and_stages_nothing(am):
    T = T_OCT + 4 * HOUR
    with am.Sweep(capacity=16) as s:
        s.set_hold_in_flight(True)
        good = timeout_cases.rec(am, 30, repeat_after_sec=60, finished_at=T - 100)
        bad = timeout_cases.rec(am, -1, repeat_after_sec=60, finished_at=T - 100)
        before = s.launch_count
        with pytest.raises(am.AmError) as e:
            s.upsert([0, 1], np.concatenate([good, bad]))
        assert e.value.code == am.AM_E_RANGE
        assert s.size == 0 and len(s.tick(T)[0]) == 0
        assert s.launch_count - before == 0  # nothing staged: no drain, and an empty shard launches nothing
        assert len(s.last_timed_out()[0]) == 0


def test_with_the_hold_off_timeouts_are_inert(am, zmap):
    n = 3000
    T = T_OCT + 9 * HOUR - 2
    rng = np.random.default_rng(9)
    recs = am.columns_to_records(population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY))))
    with am.Sweep(capacity=n) as a, am.Sweep(capacity=n) as b:
        a.upsert(np.arange(n), recs)
        recs["wf_timeout"] = rng.integers(1, 30, n)
        b.upsert(np.arange(n), recs)
        for step in [0, 1, 40, 1, 60, 3600]:
            T += step
            ga, gb = a.tick(T), b.tick(T)
            assert ga[2] == gb[2]
            np.testing.assert_array_equal(ga[0], gb[0])
            np.testing.assert_array_equal(ga[1], gb[1])
            assert len(b.last_timed_out()[0]) == 0
        da, db = a.read_range(0, n), b.read_range(0, n)
        for name in am.COLUMN_NAMES:
            np.testing.assert_array_equal(da[name], db[name], err_msg=name)


def test_launch_counts(am):
    """a handle that never receives a non-zero wf_timeout launches what it launched before timeouts existed; one that
    does launches one expiry pass per tick and one store per drain with state ops"""
    n = 64
    T = T_OCT + 3 * HOUR + 7
    rec = timeout_cases.rec
    with am.Sweep(capacity=n) as a, am.Sweep(capacity=n) as b:
        for s in (a, b):
            s.set_hold_in_flight(True)
        a.upsert(np.arange(n), np.repeat(rec(am, 0, repeat_after_sec=60, finished_at=T - 100), n))
        la, lb = a.launch_count, b.launch_count
        b.upsert(np.arange(n), np.repeat(rec(am, 30, repeat_after_sec=60, finished_at=T - 100), n))
        da, db = [], []
        for k, t in enumerate([T, T + 1, T + 30, T + 31, T + 90]):
            if k == 3:
                for s in (a, b):
                    s.upsert([3], rec(am, 0, repeat_after_sec=60, finished_at=T - 100))
                    s.post_result([4], [am.PHASE_SUCCEEDED])
            a.tick(t)
            b.tick(t)
            da.append(a.launch_count - la)
            db.append(b.launch_count - lb)
            la, lb = a.launch_count, b.launch_count
        # b: allocation (one fill) + store at the first drain, one expiry pass every tick, a store at the drain of k == 3
        assert [y - x for x, y in zip(da, db)] == [3, 1, 1, 2, 1], (da, db)
        # a: the hold-in-flight tick of before: drain (mark, state, planes, clear since, clear marks) + sweep, scan,
        # expand, publish; no drain without staged calls
        assert da[1] == da[2] == da[4] == 4, da


# ---- 5. full size, on the GPU only --------------------------------------------------------------------------------------
def test_full_size_config2_with_a_burst_of_expiries(am, zmap):
    if emulated(am):
        pytest.skip("10 M records: GPU only")
    n = 10_000_000
    T0 = amgen.T0_MON_0915
    cols = amgen.fill(2, 2, 0, n, T0, am.load().am_healthcheck_classify)
    p = Pair(am, zmap, cols, hold=True)
    rng = np.random.default_rng(2)
    try:
        recs = am.columns_to_records(cols)
        recs["wf_timeout"] = rng.integers(30, 600, n)
        p.upsert(np.arange(n), recs)
        T = T0
        for k, step in enumerate([0, 1, 59, 1, 60, 3600]):
            T += step
            if k == 3:
                fl = np.flatnonzero(p.m.since != NONE)
                sl = rng.choice(fl, min(len(fl), 50_000), replace=False)
                p.post(sl, rng.integers(1, 3, len(sl)).astype(np.uint8))
            got = p.tick(T, mode=CATCH if k == 4 else 0, entry="tick_view" if k % 2 else "tick")
            if k == 5:  # every run still held past its deadline times out at once
                assert len(got[3][0]) > 1_000_000, len(got[3][0])
    finally:
        p.close()
