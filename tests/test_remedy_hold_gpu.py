"""The remedy hold (am_sweep_set_hold_remedy, with the hold in flight on): a check is not submitted while its remedy
workflow runs, and a remedy that outlives its workflow timeout is failed on the device.  Compared after every tick with
the model (tests/handle_model.py, tests/handle_pair.py) — list, statistics, all sixteen columns, am_sweep_in_flight,
am_sweep_remedy_in_flight and both timed-out lists — through every tick entry point: the hand-derived cases, long random
sequences on the adversarial population with sparse and dense posts, catch-up ticks on named zones, next_due against
brute force, short buffers, launch counts, and 10 M records."""
import zlib

import numpy as np
import pytest

import amgen
import remedy_hold_cases
import remedy_hold_oracle
from adversarial import ZoneMap, population, zones_usable
from handle_pair import Pair, emulated

pytestmark = pytest.mark.gpu

DAY, HOUR = 86400, 3600
T_OCT = 1790812800  # 2026-10-01 00:00:00 UTC
NONE = remedy_hold_oracle.NONE
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
@pytest.mark.parametrize("case", remedy_hold_cases.CASES, ids=lambda c: c.__name__)
def test_hand_derived_cases(am, zmap, case, entry):
    p = Pair(am, zmap, _empty(am, 8), hold=True, remedy=True, entry=entry)
    try:
        case(am, p)
    finally:
        p.close()


# ---- 2. long random sequences on the adversarial population, sparse and dense posts -------------------------------------
STEPS = [1, 1, 1, 57, 1, 1, 60, 2, 1, -60, 0, 1, 17, 1, 1, 59, 1, 0, 1, 600, 1, 1, 43, 1, -1, 1, 120, 1, 1, 30, 1, 29, 1,
         3600 + 17, 1, 1, 5, 55, 1]


def _records(am, rng, n, T, zmap, wmax):
    recs = am.columns_to_records(population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))))
    recs["wf_timeout"] = np.where(rng.random(n) < 0.2, 0, rng.integers(1, wmax, n))
    return recs


def _random_walk(am, p, rng, n, T, mode, population_of):
    sl = np.arange(n)
    p.upsert(sl, population_of(n))
    for k, step in enumerate(STEPS):
        if k:
            r = rng.random()
            if r < 0.25:
                sl = rng.choice(n, 60, replace=False)
                p.upsert(sl, population_of(60))
            elif r < 0.33:
                p.remove(rng.choice(n, 30, replace=False))
            elif r < 0.41:
                first = int(rng.integers(0, n - 200))
                p.load(first, am.records_to_columns(population_of(200)))
            elif r < 0.44:
                p.set_hold(False)
                p.set_hold(True)
                p.set_remedy(True)
            elif r < 0.47:
                p.set_remedy(False)
                p.set_remedy(True)
            busy = np.flatnonzero((p.m.since != NONE) | (p.m.rsince != NONE))
            if len(busy) and k % 2:
                dense = k % 5 == 3
                sl = rng.choice(busy, min(len(busy), 2000 if dense else 30), replace=False)
                if dense:  # over an eighth of the records: applied inside the sweep
                    sl = np.concatenate([sl, rng.choice(n, 500, replace=False)])
                ph = np.where(rng.random(len(sl)) < 0.6, 2, rng.integers(0, 3, len(sl))).astype(np.uint8)
                rp = np.where(rng.random(len(sl)) < 0.5, 0, rng.integers(1, 3, len(sl))).astype(np.uint8)
                p.post(sl, ph, rp)
        T += step
        p.tick(T, mode)


@pytest.mark.parametrize("mode", [0, FULL, CATCH, CATCH | FULL], ids=["plain", "full_scan", "catch_up", "catch_up_full"])
@pytest.mark.parametrize("entry", ENTRIES + ["short_buffer"])
def test_random_sequences_equal_the_oracle(am, zmap, entry, mode):
    n = 3000
    rng = np.random.default_rng(zlib.crc32(f"remedy hold {entry} {mode}".encode()))
    T = T_OCT + 12 * DAY + 14 * HOUR - 3
    cols = population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY)))
    p = Pair(am, zmap, cols, hold=True, remedy=True, entry="tick_short" if entry == "short_buffer" else entry, cap=5)
    try:
        _random_walk(am, p, rng, n, T, mode, lambda m: _records(am, rng, m, T, zmap, 120))
        assert p.started > 100 and p.rtimed_total > 10, (p.started, p.rtimed_total)
    finally:
        p.close()


# ---- 3. catch-up ticks on named zones (amgen config 22) -------------------------------------------------------------------
def test_catch_up_on_named_zones(am, zmap):
    n = 20_000
    T = amgen.T0_MON_0915
    cols = amgen.fill(22, 2, 0, n, T, am.load().am_healthcheck_classify)
    rng = np.random.default_rng(22)
    cols["flags"] |= np.where(rng.random(n) < 0.5, am.F_HAS_REMEDY, 0).astype(np.uint32)
    p = Pair(am, zmap, cols, hold=True, remedy=True)
    try:
        recs = am.columns_to_records(cols)
        recs["wf_timeout"] = rng.integers(0, 400, n)
        p.upsert(np.arange(n), recs)
        for k, step in enumerate([0, 60, 1, 150, 59, 600, 1, 3600, 61, 240]):
            T += step
            busy = np.flatnonzero((p.m.since != NONE) | (p.m.rsince != NONE))
            if k and len(busy):
                sl = rng.choice(busy, min(len(busy), 1500), replace=False)
                p.post(sl, np.where(rng.random(len(sl)) < 0.7, 2, 0).astype(np.uint8),
                       np.where(rng.random(len(sl)) < 0.3, 1, 0).astype(np.uint8))
            p.tick(T, CATCH, entry=ENTRIES[k % 4])
        assert p.started > 100, p.started
    finally:
        p.close()


# ---- 4. next_due counts remedy deadlines and skips remedy runs --------------------------------------------------------------
def test_next_due_against_brute_force(am, zmap):
    T = T_OCT + 10 * HOUR + 20
    rec = remedy_hold_cases.rec
    recs = np.concatenate([rec(am, 45, repeat_after_sec=600, finished_at=T - 1000, has_remedy=True),
                           rec(am, 7, repeat_after_sec=60, finished_at=T - 5000, has_remedy=True),
                           rec(am, 0, repeat_after_sec=300, finished_at=T - 1000, has_remedy=True),
                           rec(am, 200, cron="*/5 * * * *", has_remedy=True),
                           rec(am, 90, cron="7 * * * *")])
    p = Pair(am, zmap, _empty(am, len(recs)), hold=True, remedy=True)
    try:
        p.upsert(np.arange(len(recs)), recs)
        checked = 0
        for step, post in [(0, None), (1, [0, 1, 2, 3]), (3, None), (5, None), (30, [2]), (1, None), (200, [3])]:
            T += step
            if post:
                p.post(post, [2] * len(post))
            p.tick(T)
            assert p.s.next_due(T) == p.m.first_active_tick(T, 4000), T
            checked += 1
        assert checked == 7 and p.started >= 3
    finally:
        p.close()


# ---- 5. launch counts --------------------------------------------------------------------------------------------------------
def test_launch_counts(am):
    """the remedy hold adds no launch to a tick (its sweep and result kernels replace the hold's); turning it off is one
    pass over the slots; a handle without it launches what it launched before"""
    n = 64
    T = T_OCT + 3 * HOUR + 7
    rec = remedy_hold_cases.rec
    with am.Sweep(capacity=n) as a, am.Sweep(capacity=n) as b:
        for s in (a, b):
            s.set_hold_in_flight(True)
        b.set_hold_remedy(True)
        for s in (a, b):
            s.upsert(np.arange(n), np.repeat(rec(am, 30, repeat_after_sec=60, finished_at=T - 100, has_remedy=True), n))
        la, lb = a.launch_count, b.launch_count
        da, db = [], []
        for k, t in enumerate([T, T + 1, T + 30, T + 31, T + 50]):
            if k in (1, 3):
                for s in (a, b):
                    s.post_result([4], [2])
            a.tick(t)
            b.tick(t)
            da.append(a.launch_count - la)
            db.append(b.launch_count - lb)
            la, lb = a.launch_count, b.launch_count
        assert da == db, (da, db)
        # a: the timeout tick of before: (allocation + store) + drain + expiry + sweep, scan, expand, publish
        assert da[2] == da[4] == 5 and da[0] == 12, da
        assert b.remedy_in_flight(0, n)[4] != NONE
        lb = b.launch_count
        b.set_hold_remedy(False)
        assert b.launch_count - lb == 1 and (b.remedy_in_flight(0, n) == NONE).all()


# ---- 6. full size, on the GPU only ----------------------------------------------------------------------------------------
def test_full_size_config3(am, zmap):
    if emulated(am):
        pytest.skip("10 M records: GPU only")
    n = 10_000_000
    T0 = amgen.T0_MON_0915
    cols = amgen.fill(3, 3, 0, n, T0, am.load().am_healthcheck_classify)
    p = Pair(am, zmap, cols, hold=True, remedy=True)
    rng = np.random.default_rng(3)
    try:
        recs = am.columns_to_records(cols)
        recs["wf_timeout"] = rng.integers(30, 600, n)
        p.upsert(np.arange(n), recs)
        T = T0
        for k, step in enumerate([0, 1, 59, 1, 60, 3600]):
            T += step
            if k in (1, 3):
                fl = np.flatnonzero(p.m.since != NONE)
                sl = rng.choice(fl, min(len(fl), 50_000 if k == 1 else 2_000_000), replace=False)
                p.post(sl, np.full(len(sl), 2, dtype=np.uint8))
            p.tick(T, mode=CATCH if k == 4 else 0, entry="tick_view" if k % 2 else "tick")
        assert p.started > 100_000 and p.rtimed_total > 10_000, (p.started, p.rtimed_total)
    finally:
        p.close()
