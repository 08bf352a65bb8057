"""Hold in flight (am_sweep_set_hold_in_flight): a check whose health-check workflow is running is not submitted again
until a workflow phase is posted for it, it is removed or its slot is loaded.  Compared after every tick with the hold
oracle (tests/hold_oracle.py, through tests/handle_pair.py) — list, statistics, all sixteen columns and
am_sweep_in_flight — and checked against an
invariant that needs no oracle, the release / clear / keep cases, the refusals, short buffers, turning the hold off
and next_due."""
import zlib

import numpy as np
import pytest

import amgen
import hold_oracle
from adversarial import ZoneMap, population, zones_usable
from handle_pair import Pair, emulated

pytestmark = pytest.mark.gpu

DAY, HOUR = 86400, 3600
T_OCT = 1790812800  # 2026-10-01 00:00:00 UTC
NONE = hold_oracle.NOT_IN_FLIGHT
FULL, CATCH = 0x2, 0x8


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def _past(cols, T):
    """no finishedAt after T: a check finishes before a controller sees it"""
    cols["finished_at"][:] = np.minimum(cols["finished_at"], T)
    return cols


def _records(am, rng, n, T, zmap):
    return am.columns_to_records(population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY))))


# ---- 1. tens of ticks with calls in between, every entry point, against the hold oracle -----------------------------
# (-60 and 0: a wall clock stepped back and a second ticked twice — a posted phase releases the hold all the same)
STEPS = [1, 1, 1, 57, 1, 1, 60, 2, 1, -60, 0, 1, 3600 + 17, 1, 1, 59, 1, 0, 1, 600, 1, 1, 43, 1, -1, 1, 120, 1, 1]


@pytest.mark.parametrize("mode", [0, FULL, CATCH, CATCH | FULL], ids=["plain", "full_scan", "catch_up", "catch_up_full"])
@pytest.mark.parametrize("entry", ["tick", "tick_view", "tick_device", "tick_shard"])
def test_ticks_equal_the_hold_oracle(am, zmap, entry, mode):
    n = 3000
    rng = np.random.default_rng(zlib.crc32(f"{entry} {mode}".encode()))
    T = T_OCT + 12 * DAY + 14 * HOUR - 3
    p = Pair(am, zmap, population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))), hold=True, entry=entry)
    held_seen = released = superseded = 0
    try:
        for k, step in enumerate(STEPS):
            if k:
                # calls staged between ticks
                r = rng.random()
                if r < 0.3:
                    sl = rng.choice(n, 40, replace=False)
                    p.upsert(sl, _records(am, rng, 40, T, zmap))
                elif r < 0.45:
                    p.remove(rng.choice(n, 30, replace=False))
                elif r < 0.55:
                    first = int(rng.integers(0, n - 200))
                    p.load(first, population(rng, 200, T, True, zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))))
                fl = np.flatnonzero(p.m.since != NONE)
                if len(fl):
                    dense = k % 5 == 3
                    sl = rng.choice(fl, min(len(fl), 2000 if dense else 40), replace=False)
                    if dense:  # over an eighth of the records: applied inside the sweep
                        sl = np.concatenate([sl, rng.choice(n, 500, replace=False)])
                    p.post(sl, rng.integers(1, 3, len(sl)), rng.integers(0, 3, len(sl)).astype(np.uint8))
                    released += len(sl)
                    if k % 3 == 1:  # an upsert of posted slots in the same drain: it supersedes the result, not the release
                        up = sl[:10]
                        p.upsert(up, _records(am, rng, len(up), T, zmap))
                        superseded += len(up)
                if k % 4 == 2:  # a read's drain: the results stay pending for the sweep
                    np.testing.assert_array_equal(p.s.in_flight(0, n), p.m.in_flight())
            T += step
            held_seen += int(p.m.held().sum())
            p.tick(T, mode)
        assert held_seen > 1000 and released > 100 and superseded > 30
    finally:
        p.close()


# ---- 2. the invariant: one submission per run, no oracle ---------------------------------------------------------
@pytest.mark.parametrize("with_results", [False, True])
def test_no_second_submission_while_in_flight(am, zmap, with_results):
    n = 2000
    ticks = 600 if emulated(am) else 3600
    rng = np.random.default_rng(17 + with_results)
    T0 = T_OCT + 5 * DAY + 9 * HOUR + 13
    cols = _past(population(rng, n, T0, True, zmap.ids_of(zones_usable(T0 - DAY, T0 + DAY))), T0)
    kind = cols["flags"] & np.uint32(am.KIND_MASK)
    with am.Sweep(capacity=n) as s:
        s.set_hold_in_flight(True)
        s.load_range(0, cols)
        allowed = np.ones(n, dtype=bool)  # may be submitted (nothing in flight since the last release)
        count = np.zeros(n, dtype=np.int64)
        for t in range(ticks):
            idx, act, _ = s.tick_view(T0 + t)
            sub = idx[(act & am.ACT_SUBMIT_HC) != 0].astype(np.int64)
            assert allowed[sub].all(), (t, sub[~allowed[sub]][:5])
            allowed[sub] = False
            count[sub] += 1
            if with_results and t % 7 == 3:
                busy = np.flatnonzero(~allowed)
                if len(busy):
                    sl = rng.choice(busy, min(len(busy), 60), replace=False)
                    s.post_result(sl, rng.integers(1, 3, len(sl)).astype(np.uint8))
                    allowed[sl] = True
        sched = (kind == am.KIND_INTERVAL) | (kind == am.KIND_CRON_EVERY) | (kind == am.KIND_CRON_SPEC)
        if not with_results:
            assert count.max() <= 1
            assert count[sched].sum() > n // 5
        else:
            assert count.max() >= 2


# ---- 3. release, clear and keep ----------------------------------------------------------------------------------
def _interval(am, n, fa):
    rc, r = am.classify(repeat_after_sec=1, finished_at=fa)
    assert rc == 0
    return np.repeat(r, n)


@pytest.mark.parametrize("route", ["drain_kernel", "sweep", "read_drain"])
def test_a_posted_phase_releases_the_hold(am, route):
    n = 64
    T = T_OCT + 3 * HOUR + 7
    with am.Sweep(capacity=n) as s:
        s.set_hold_in_flight(True)
        s.upsert(np.arange(n), _interval(am, n, T - 100))
        idx, _, _ = s.tick(T)
        assert len(idx) == n and (s.in_flight(0, n) == T).all()
        assert len(s.tick(T + 1)[0]) == 0  # due by the timer, held
        sl = [5] if route != "sweep" else np.arange(n)  # one result: the drain kernel; all of them: the sweep
        s.post_result(sl, np.full(len(sl), am.PHASE_FAILED, np.uint8))
        if route == "read_drain":
            assert s.in_flight(idx=[5])[0] == NONE  # drained by the read: left pending, released
        before = s.launch_count
        idx, _, st = s.tick(T + 2)  # applies the result: finishedAt = T + 2, timer re-armed for a second
        assert st["n_result_fail"] == len(sl) and len(idx) == 0
        assert s.in_flight(0, n)[5] == NONE
        assert s.launch_count > before
        idx, _, _ = s.tick(T + 3)
        assert sorted(idx.tolist()) == sorted(np.asarray(sl).tolist())
        assert s.in_flight(idx=[5])[0] == T + 3


@pytest.mark.parametrize("case", ["upsert_after_post", "clock_back", "same_second", "remedy_only"])
def test_a_posted_phase_releases_whatever_follows_it(am, case):
    """the release happens at the drain: an upsert that supersedes the result itself (staged calls take effect in call
    order), or a tick second not later than the submission, does not keep the check held; a remedy phase alone does"""
    n = 16
    T = T_OCT + 5 * HOUR + 11
    with am.Sweep(capacity=n) as s:
        s.set_hold_in_flight(True)
        s.upsert(np.arange(n), _interval(am, n, T - 100))
        assert len(s.tick(T)[0]) == n
        if case == "remedy_only":
            s.post_result([5], [am.PHASE_NONE], [am.PHASE_SUCCEEDED])
        else:
            s.post_result([5], [am.PHASE_SUCCEEDED])
        if case == "upsert_after_post":  # the informer's pre-run record: finishedAt T - 100 <= since
            s.upsert([5], _interval(am, 1, T - 100))
        T1 = {"upsert_after_post": T + 1, "clock_back": T - 60, "same_second": T, "remedy_only": T + 1}[case]
        subs = []
        for t in range(T1, T1 + 30):
            idx, act, _ = s.tick(t)
            subs += [t for i, a in zip(idx.tolist(), act.tolist()) if i == 5 and a & am.ACT_SUBMIT_HC]
        if case == "remedy_only":
            assert subs == [] and s.in_flight(idx=[5])[0] == T
        else:
            # submitted once, at the first second its timer allows, and held from then on
            first = T1 if case == "upsert_after_post" else T1 + 1
            assert subs == [first], subs
            assert s.in_flight(idx=[5])[0] == first
        assert (s.in_flight(idx=[4, 6]) == T).all()


def test_remove_upsert_and_load_clear_or_keep(am):
    n = 16
    T = T_OCT + 4 * HOUR
    with am.Sweep(capacity=n) as s:
        s.set_hold_in_flight(True)
        s.upsert(np.arange(n), _interval(am, n, T - 100))
        assert len(s.tick(T)[0]) == n
        s.remove([2])
        assert len(s.tick(T + 1)[0]) == 0
        s.upsert([2], _interval(am, 1, T - 100))            # clear: remove and upsert, two drains
        s.remove([0])                                       # clear: remove
        s.remove([1])
        s.upsert([1], _interval(am, 1, T - 100))            # clear: remove, then upsert, one drain
        s.upsert([3], _interval(am, 1, T - 100))            # keep: an upsert alone (a status write during the run)
        s.upsert([4], _interval(am, 1, T - 5000))           # keep: an upsert with an earlier finishedAt
        s.upsert([5], _interval(am, 1, T + 1))              # release: finishedAt later than since
        cols = am.records_to_columns(_interval(am, 2, T - 100))
        s.load_range(6, cols)                               # clear: load_range
        f = s.in_flight(0, n)
        np.testing.assert_array_equal(s.in_flight(), f)  # (default: every swept slot)
        assert f[0] == NONE and f[1] == NONE and f[2] == NONE and f[5] == NONE and f[6] == NONE and f[7] == NONE
        assert f[3] == T and f[4] == T and (f[8:] == T).all()
        idx, _, _ = s.tick(T + 2)
        assert sorted(idx.tolist()) == [1, 2, 5, 6, 7]


def test_a_stopped_report_releases_the_hold(am):
    T = T_OCT + 6 * HOUR
    with am.Sweep(capacity=8) as s:
        s.set_hold_in_flight(True)
        s.upsert([0], _interval(am, 1, T - 100))
        assert s.tick(T)[0].tolist() == [0]
        rc, stopped = am.classify(repeat_after_sec=0, finished_at=T - 100)
        assert rc == 0 and stopped["flags"][0] & am.KIND_MASK == am.KIND_STOPPED
        s.upsert([0], stopped)  # paused during the run: keeps since (finishedAt T - 100 <= since) ...
        assert s.in_flight(idx=[0])[0] == T
        idx, act, _ = s.tick(T + 1)  # ... until the pause is reported: finishedAt = T + 1
        assert idx.tolist() == [0] and act.tolist() == [am.ACT_STOPPED]
        assert s.in_flight(idx=[0])[0] == NONE
        s.upsert([0], _interval(am, 1, T + 1))  # resumed with the status the report wrote
        assert s.tick(T + 3)[0].tolist() == [0]


# ---- 4. refusals -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("entry", ["tick", "tick_view", "tick_device", "tick_shard", "run_ticks", "run_ticks_blocked"])
def test_closed_loop_and_run_ticks_are_refused_without_effect(am, entry):
    n = 32
    T = T_OCT + 7 * HOUR + 30
    with am.Sweep(capacity=n) as s:
        s.set_hold_in_flight(True)
        s.upsert(np.arange(n), _interval(am, n, T - 100))
        s.tick(T)
        s.post_result([3], [am.PHASE_SUCCEEDED])
        s.upsert([4], _interval(am, 1, T + 5))
        before = s.launch_count
        with pytest.raises(am.AmError) as e:
            if entry == "tick":
                s.tick(T + 1, mode=am.SWEEP_CLOSED_LOOP)
            elif entry == "tick_view":
                s.tick_view(T + 1, mode=am.SWEEP_CLOSED_LOOP)
            elif entry == "tick_device":
                s.tick_device(T + 1, am.SWEEP_CLOSED_LOOP, 0, 0, 0, 0, 0)
            elif entry == "tick_shard":
                s.tick_shard(T + 1, mode=am.SWEEP_CLOSED_LOOP)
            else:
                s.run_ticks(T + 1, 5, mode=am.SWEEP_BLOCKED if entry == "run_ticks_blocked" else 0)
        assert e.value.code == am.AM_E_INVAL
        assert s.launch_count == before  # nothing drained, nothing launched
        with pytest.raises(am.AmError) as e:  # P unchanged: a day and a second after T is still refused
            s.tick(T + DAY + 1, mode=am.SWEEP_CATCH_UP)
        assert e.value.code == am.AM_E_RANGE
        f = s.in_flight(0, n)  # the staged calls are still there
        assert f[3] == NONE and f[4] == NONE and f[5] == T
        s.set_hold_in_flight(False)
        s.tick(T + 2, mode=am.SWEEP_CLOSED_LOOP)


# ---- 5. short buffers; turning the hold off ----------------------------------------------------------------------
def test_a_short_buffer_tick_holds_the_whole_list(am, zmap):
    n = 3000
    T = T_OCT + 8 * HOUR
    rng = np.random.default_rng(8)
    with am.Sweep(capacity=n) as s:
        s.set_hold_in_flight(True)
        s.load_range(0, _past(population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY))), T))
        with pytest.raises(am.AmError) as e:
            s.tick(T, cap=3)
        assert e.value.code == am.AM_E_NOSPACE
        idx, act, left = s.last_list(0, n)
        assert left == e.value.needed > 100
        sub = np.zeros(n, bool)
        sub[idx[(act & am.ACT_SUBMIT_HC) != 0].astype(np.int64)] = True
        f = s.in_flight(0, n)
        assert (f[sub] == T).all() and (f[~sub] == NONE).all()
        idx, act, _ = s.tick(T + 1)
        assert not sub[idx[(act & am.ACT_SUBMIT_HC) != 0].astype(np.int64)].any()


def test_hold_on_then_off_ticks_like_never_on(am, zmap):
    n = 3000
    T = T_OCT + 9 * HOUR - 2
    rng = np.random.default_rng(9)
    cols = population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY)))
    with am.Sweep(capacity=n) as a, am.Sweep(capacity=n) as b:
        for s in (a, b):
            s.load_range(0, cols)
        b.set_hold_in_flight(True)
        b.tick(T)
        b.set_hold_in_flight(False)
        a.tick(T)
        assert (b.in_flight(0, n) == NONE).all()
        for k, step in enumerate([1, 1, 1, 60, 1, 61, 3600]):
            T += step
            for s in (a, b):
                s.post_result(np.arange(k, n, 23), np.full(len(range(k, n, 23)), am.PHASE_SUCCEEDED, np.uint8))
                s.remove([k + 1])
            la, lb = a.launch_count, b.launch_count
            ga = a.tick(T, mode=CATCH if k % 2 else 0)
            gb = b.tick(T, mode=CATCH if k % 2 else 0)
            assert a.launch_count - la == b.launch_count - lb, k
            assert ga[2] == gb[2]
            np.testing.assert_array_equal(ga[0], gb[0])
            np.testing.assert_array_equal(ga[1], gb[1])
        da, db = a.read_range(0, n), b.read_range(0, n)
        for name in am.COLUMN_NAMES:
            np.testing.assert_array_equal(da[name], db[name], err_msg=name)


# ---- 6. next_due skips held records --------------------------------------------------------------------------------
def test_next_due_is_the_first_tick_that_emits(am, zmap):
    T = T_OCT + 10 * HOUR + 20
    specs = [dict(repeat_after_sec=r, finished_at=T - d) for r, d in [(30, 100), (45, 10), (90, 200), (120, 5), (7, 1)]]
    specs += [dict(cron=c) for c in ["*/3 * * * *", "7 * * * *", "CRON_TZ=Asia/Kathmandu * * * * *"]]
    recs = np.concatenate([am.classify(**kw)[1] for kw in specs])
    n = len(recs)
    cols = am.records_to_columns(recs)
    p = Pair(am, zmap, cols, hold=True)
    try:
        for k, (step, post) in enumerate([(0, None), (1, None), (13, [0]), (1, None), (200, [1, 2]), (1, None)]):
            T += step
            if post:
                p.post(post, [am.PHASE_SUCCEEDED] * len(post))
            p.tick(T)
            nd = p.s.next_due(T)
            t = p.m.first_active_tick(T, 4000)  # (no result is pending: the first tick that emits)
            assert t is not None and nd == t, (k, nd, t)
    finally:
        p.close()


@pytest.mark.parametrize("parse_errors", [True, False])
def test_next_due_on_the_adversarial_population(am, zmap, parse_errors):
    """next_due against oracle ticks one second at a time, on adversarial records with zones, some of them held
    STOPPED / PARSE_ERROR records (in flight when the CR was paused or broken).  No tick before next_due emits; next_due
    itself emits, unless it is the next UTC minute standing in for a zone-bound schedule (a lower bound by design)."""
    n = 400
    T = T_OCT + 11 * HOUR + 7
    rng = np.random.default_rng(31 + parse_errors)
    cols = population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY)))
    if not parse_errors:  # (a PARSE_ERROR record is due every second: next_due would always be T + 1)
        pe = (cols["flags"] & np.uint32(am.KIND_MASK)) == am.KIND_PARSE_ERROR
        cols["flags"][pe] = am.F_TOMBSTONE
    p = Pair(am, zmap, cols, hold=True)
    checked = 0
    try:
        for k, step in enumerate([0, 1, 1, 29, 1, 1, 61]):
            T += step
            if k == 2:  # paused / broken during their runs: held STOPPED and PARSE_ERROR records
                sub = np.flatnonzero(p.m.since != NONE)[:6]
                assert len(sub) == 6
                rc, stopped = am.classify(repeat_after_sec=0, finished_at=T - 3)
                rc2, broken = am.classify(cron="bad cron", finished_at=T - 3)
                assert stopped["flags"][0] & am.KIND_MASK == am.KIND_STOPPED
                assert broken["flags"][0] & am.KIND_MASK == am.KIND_PARSE_ERROR
                recs = np.concatenate([stopped] * 3 + [broken if parse_errors else stopped] * 3)
                p.upsert(sub, recs)
                assert p.m.held()[sub].all()
            if k == 4:
                fl = np.flatnonzero(p.m.since != NONE)
                p.post(fl[::3], np.full(len(fl[::3]), am.PHASE_SUCCEEDED, np.uint8))
            got = p.tick(T)
            if k == 2:  # held, and still reported
                acts = dict(zip(got[0].tolist(), got[1].tolist()))
                assert all(acts.get(int(i), 0) & (am.ACT_STOPPED | am.ACT_PARSE_ERROR) for i in sub)
            nd = p.s.next_due(T)
            oc = {kk: v.copy() for kk, v in p.m.cols().items()}
            since = p.m.since.copy()
            t = T + 1
            while nd is None or t < min(nd, T + 3600):
                assert len(hold_oracle.sweep(zmap, oc, since, t)[0]) == 0, (k, t, nd)
                t += 1
                if nd is None and t > T + 3600:
                    break
            if nd is not None and nd <= T + 3600:
                f = oc["flags"]
                zone_cron = ((f & np.uint32(am.KIND_MASK)) == am.KIND_CRON_SPEC) & ((f >> np.uint32(24)) != 0) & \
                            ((f & np.uint32(am.F_TOMBSTONE)) == 0) & ~hold_oracle.held(oc, since)
                emits = len(hold_oracle.sweep(zmap, oc, since, nd)[0]) > 0
                assert emits or (nd % 60 == 0 and zone_cron.any()), (k, nd)
                checked += 1
        assert checked >= 5
    finally:
        p.close()


# ---- 7. full size, on the GPU only ---------------------------------------------------------------------------------
def test_full_size_config2_against_the_oracle(am, zmap):
    if emulated(am):
        pytest.skip("10 M records: GPU only")
    n = 10_000_000
    T0 = amgen.T0_MON_0915
    cols = amgen.fill(2, 2, 0, n, T0, am.load().am_healthcheck_classify)
    p = Pair(am, zmap, cols, hold=True)
    rng = np.random.default_rng(2)
    try:
        T = T0
        for k, step in enumerate([0, 1, 59, 1, 60]):
            T += step
            if k == 3:
                fl = np.flatnonzero(p.m.since != NONE)
                sl = rng.choice(fl, min(len(fl), 50_000), replace=False)
                p.post(sl, rng.integers(1, 3, len(sl)).astype(np.uint8))
            p.tick(T, mode=CATCH if k == 4 else 0, entry="tick_view" if k % 2 else "tick")
    finally:
        p.close()
