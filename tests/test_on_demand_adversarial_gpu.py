"""The on-demand queries and the hold sweep variants at adversarial records and instants, against the C oracle:
am_sweep_repeat_after_sec on the adversarial population (tests/adversarial.py) in and beyond the library's domain, at
every instant of TS and at leap-day, year-end and five-year give-up instants, over ragged sub-ranges, behind staged
upserts and removes and at a shard base past 2^32; am_sweep_next_due, exactly, on quiet populations whose next event is
minutes to years away, with the hold, workflow timeouts and remedy runs, and over 10 M records with one winner; and
random walks of the hold, hold + timeouts, remedy hold and remedy hold + timeouts at every instant of TS."""
import ctypes as C
import os
import zlib

import numpy as np
import pytest

import amgen
import oracle_c
import test_remedy_hold_gpu
from adversarial import I32MAX, I32MIN, TS, ZoneMap, population, zones_usable
from handle_pair import Pair

pytestmark = pytest.mark.gpu

DAY = 86400
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
NONE = INT64_MIN                # no run in flight (hold_oracle.NOT_IN_FLIGHT)
NO_DEADLINE = INT64_MAX         # (timeout_oracle.NO_DEADLINE)
SATURATED = -9223372035         # RepeatAfterSec when Next() finds nothing within five years
MASKS = ("minute", "hour", "dom", "month", "dow")
FULL, CATCH = 0x2, 0x8

LEAP_2000_END = 951868799       # 2000-02-29 23:59:59
END_2099 = 4102444799           # 2099-12-31 23:59:59
FEB28_2100_END = 4107542399     # 2100-02-28 23:59:59 (2100 is not a leap year: March follows)
LEAP_2096 = 3981312000          # 2096-02-29 00:00:00: the next Feb 29 (2104) is past 2096 + 5
GIVE_UP_LAST = 4070908798       # 2098-12-31 23:59:58: "0 0 29 2 *" gives up (2104 > 2098 + 5) ...
GIVE_UP_FOUND = 4070908799      # ... and a second later Next() starts in 2099 and finds 2104-02-29
FEB29_2104 = 4233686400         # 2104-02-29 00:00:00
EDGES = [LEAP_2000_END, END_2099, FEB28_2100_END, LEAP_2096, GIVE_UP_LAST, GIVE_UP_FOUND]
INSTANTS = TS + EDGES
LORD_HOWE = "Australia/Lord_Howe"  # daylight saving time of half an hour


def _tid(T):
    return f"T={T}"


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def _emulated(am):
    return "emu" in os.path.basename(am.abi.LIB_PATH)


def _orc_cron(cols, i, tz_id=0):
    return oracle_c.OrcCron(*(int(cols[m][i]) for m in MASKS), 0, 1, tz_id)


# ---- 1. am_sweep_repeat_after_sec --------------------------------------------------------------------------------------
def _repeat_after_want(am, lib, zmap, cols, T):
    """the rule of include/amsweep.h per record: 0 for a tombstone and the kinds without a schedule, the stored interval
    (whatever its sign) for INTERVAL / CRON_EVERY, Next(T) - T of the oracle for CRON_SPEC (its zone id translated)"""
    f = cols["flags"]
    kind = f & np.uint32(am.KIND_MASK)
    live = (f & np.uint32(am.F_TOMBSTONE)) == 0
    want = np.zeros(len(f), dtype=np.int64)
    iv = live & ((kind == am.KIND_INTERVAL) | (kind == am.KIND_CRON_EVERY))
    want[iv] = cols["ras"][iv]
    for i in np.flatnonzero(live & (kind == am.KIND_CRON_SPEC)):
        c = _orc_cron(cols, i, int(zmap.fwd[f[i] >> np.uint32(am.F_TZ_SHIFT)]))
        want[i] = lib.orc_cron_repeat_after_sec(C.byref(c), T)
    return want


RA_SIZES = [1, 127, 129, 1023, 1025, 70_001]


@pytest.mark.parametrize("in_domain", [True, False], ids=["library-domain", "beyond-domain"])
@pytest.mark.parametrize("T", INSTANTS, ids=_tid)
def test_repeat_after_sec_equals_the_oracle(am, orc, zmap, T, in_domain):
    """Every size of RA_SIZES loaded at a ragged offset of a larger handle (every other one with a shard base past
    2^32), then upserts and removes staged: the query applies them first.  The whole loaded range and three ragged
    sub-ranges of it equal the rule, record by record."""
    lib = orc.load()
    rng = np.random.default_rng(zlib.crc32(f"repeat after {T} {in_domain}".encode()))
    # (zone-bound schedules are evaluated on the host, minute by minute: bound at the smaller sizes only.  Not Lord
    # Howe: see test_repeat_after_sec_across_a_half_hour_daylight_saving_gap)
    tz = zmap.ids_of([z for z in zones_usable(T, T + 6 * 366 * DAY) if z != LORD_HOWE])
    for k, n in enumerate(RA_SIZES):
        lead = int(rng.integers(1, 300))
        cap = lead + n + int(rng.integers(0, 200))
        bound = tz if n <= 129 else []
        cols = population(rng, n, T, in_domain, bound)
        with am.Sweep(capacity=cap, shard_base=(1 << 32) + 3 if k % 2 else 0) as s:
            s.load_range(lead, cols)
            up = rng.choice(n, min(n, 40), replace=False)
            recs = am.columns_to_records(population(rng, len(up), T, in_domain, bound))
            s.upsert(up + lead, recs)
            for j, i in enumerate(up):
                for name in am.COLUMN_NAMES:
                    cols[name][i] = recs[name][j]
                cols["flags"][i] &= np.uint32(~am.F_TOMBSTONE & 0xFFFFFFFF)
            gone = rng.choice(n, min(n, 9), replace=False)
            s.remove(gone + lead)
            cols["flags"][gone] = am.F_TOMBSTONE
            want = _repeat_after_want(am, lib, zmap, cols, T)
            np.testing.assert_array_equal(s.repeat_after_sec(T, lead, n), want, err_msg=f"n={n}")
            for _ in range(3):
                a = int(rng.integers(0, n))
                b = int(rng.integers(a + 1, n + 1))
                np.testing.assert_array_equal(s.repeat_after_sec(T, lead + a, b - a), want[a:b],
                                              err_msg=f"n={n} [{a}, {b})")


def test_repeat_after_sec_hand_cases(am, orc, zmap):
    """An interval record whose stored interval is -1 next to a schedule bound to a named zone (the host evaluates the
    latter; the former keeps -1), the other i32 extremes, Feb 29 past the five-year give-up and just inside it, Feb 30,
    and masks whose only bits are out of range (minute 60+, hour 24+, day-of-month 0, month 0 and 13+)."""
    lib = orc.load()

    def rec(**kw):
        rc, r = am.classify(**kw)
        assert rc == 0, kw
        return r

    interval = rec(repeat_after_sec=60, finished_at=0)
    every = rec(cron="@every 1m")
    assert every["flags"][0] & am.KIND_MASK == am.KIND_CRON_EVERY

    def with_ras(r, v):
        r = r.copy()
        r["ras"] = v
        return r

    def with_masks(**masks):
        r = rec(cron="* * * * *")
        for name, v in masks.items():
            r[name] = np.uint64(v)
        return r

    bound = rec(cron=f"CRON_TZ={[z for z in amgen.ZONES if z != LORD_HOWE][0]} 30 4 * * *")
    assert bound["flags"][0] >> am.F_TZ_SHIFT != 0
    cases = [  # (record, wanted at every instant or None: the oracle's answer alone)
        (with_ras(interval, -1), -1), (bound, None), (with_ras(every, -1), -1), (bound, None),
        (with_ras(interval, I32MIN), I32MIN), (with_ras(every, 0), 0), (with_ras(interval, I32MAX), I32MAX),
        (rec(cron="0 0 30 2 *"), SATURATED),
        (with_masks(minute=(1 << 60) | (1 << 61)), SATURATED), (with_masks(hour=1 << 24), SATURATED),
        (with_masks(dom=1), SATURATED), (with_masks(month=1), SATURATED), (with_masks(month=1 << 13), SATURATED),
        (rec(cron="0 0 29 2 *"), None)]
    recs = np.concatenate([r for r, _ in cases])
    n = len(recs)
    cols = am.records_to_columns(recs)
    with am.Sweep(capacity=n + 5, shard_base=(1 << 33) + 1) as s:
        s.upsert(np.arange(n) + 5, recs)
        for T in (LEAP_2096, LEAP_2096 + 1, GIVE_UP_LAST, GIVE_UP_FOUND, FEB28_2100_END, TS[0], 0):
            got = s.repeat_after_sec(T, 5, n)
            np.testing.assert_array_equal(got, _repeat_after_want(am, lib, zmap, cols, T), err_msg=str(T))
            for k, (_, v) in enumerate(cases):
                if v is not None:
                    assert got[k] == v, (T, k, got[k])
            assert 0 < got[1] <= DAY and got[1] == got[3], (T, got[1])
            feb29 = got[-1]
            if T in (LEAP_2096, LEAP_2096 + 1, GIVE_UP_LAST):
                assert feb29 == SATURATED, (T, feb29)
            elif T == GIVE_UP_FOUND:
                assert feb29 == FEB29_2104 - T, (T, feb29)
        assert s.repeat_after_sec(LEAP_2096, n + 4, 1)[0] == SATURATED  # (slot n + 4: the last hand case alone)


@pytest.mark.xfail(strict=True, raises=AssertionError,
                   reason="am_cron_next takes the first instant whose local wall clock matches; robfig's Next() steps "
                          "hours in absolute time and so keeps the half hour of Lord Howe's spring-forward gap")
def test_repeat_after_sec_across_a_half_hour_daylight_saving_gap(am, orc, zmap):
    """On 2026-10-04 Lord Howe's clocks go from 02:00 (+10:30) to 02:30 (+11).  For "0,31 3 4 10 *" robfig's Next()
    walks that day's hours from local midnight one absolute hour at a time, 01:00, 02:30, 03:30, and fires at 03:31
    (16:31 UTC); the library answers 03:00 (16:00 UTC), whose wall clock matches the schedule."""
    rc, r = am.classify(cron=f"CRON_TZ={LORD_HOWE} 0,31 3 4 10 *")
    assert rc == 0
    T = TS[0]
    want = _repeat_after_want(am, orc.load(), zmap, am.records_to_columns(r), T)[0]
    if want != 1791045060 - T:  # 2026-10-03 16:31:00 UTC
        pytest.fail(f"oracle: {want}")
    with am.Sweep(capacity=1) as s:
        s.upsert([0], r)
        assert s.repeat_after_sec(T, 0, 1)[0] == want


# ---- 2. am_sweep_next_due, exactly --------------------------------------------------------------------------------------
def _next_due_want(am, lib, cols, T, since=None, deadline=None, rsince=None, rdeadline=None, floor=None):
    """The minimum over live records of each one's next event as next_due_kernel's comment defines it: T + 1 when
    something is pending; for a held run its deadline D as max(D, floor) (floor = T + 1), nothing without one; else the
    armed repeat timer finishedAt + RepeatAfterSec when it is later than T + 1 (else T + 1), or the oracle's Next(T).
    `since` / `deadline`: the health-check runs of the hold oracles; `rsince` / `rdeadline`: the remedy runs.  Records
    bound to a named zone are not expected here.  None when nothing will ever be due."""
    floor = T + 1 if floor is None else floor
    f = cols["flags"]
    kind = f & np.uint32(am.KIND_MASK)
    live = (((np.uint32(0x3E) >> kind) & np.uint32(1)) != 0) & ((f & np.uint32(am.F_TOMBSTONE)) == 0)
    pend = (((f & np.uint32(am.F_PENDING_OK | am.F_PENDING_FAIL | am.F_REMEDY_PENDING)) != 0)
            | (kind == am.KIND_PARSE_ERROR) | ((kind == am.KIND_STOPPED) & ((f & np.uint32(am.F_STOPPED_REPORTED)) == 0)))
    due = np.full(len(f), INT64_MAX, dtype=np.int64)
    due[pend] = T + 1
    held = np.zeros(len(f), dtype=bool)
    dl = np.full(len(f), NO_DEADLINE, dtype=np.int64)
    if since is not None:
        hc = (since != NONE) & (since >= cols["finished_at"]) & ~pend
        held |= hc
        dl = np.where(hc, deadline, dl)
    if rsince is not None:
        rm = (rsince != NONE) & ~pend
        held |= rm
        dl = np.where(rm, rdeadline, dl)
    hd = held & (dl != NO_DEADLINE)
    due[hd] = np.maximum(dl[hd], floor)
    rest = ~pend & ~held
    iv = rest & ((kind == am.KIND_INTERVAL) | (kind == am.KIND_CRON_EVERY))
    at = (cols["finished_at"].view(np.uint64) + cols["ras"].astype(np.int64).view(np.uint64)).view(np.int64)
    armed = (f & np.uint32(am.F_TIMER_ARMED)) != 0
    due[iv] = np.where(armed & (at > T + 1), at, T + 1)[iv]
    cr = np.flatnonzero(rest & (kind == am.KIND_CRON_SPEC) & live)
    assert not (f[cr] >> np.uint32(am.F_TZ_SHIFT)).any()
    if len(cr):  # Next(T) once per distinct schedule
        masks, inv = np.unique(np.stack([cols[m][cr] for m in MASKS], axis=1), axis=0, return_inverse=True)
        nx = np.array([lib.orc_cron_next(C.byref(oracle_c.OrcCron(*(int(v) for v in u), 0, 1, 0)), T) for u in masks],
                      dtype=np.int64)[inv.ravel()]
        due[cr] = np.where(nx != INT64_MIN, nx, INT64_MAX)
    m = int(due[live].min()) if live.any() else INT64_MAX
    return None if m == INT64_MAX else m


def _quiet(am, rng, n, T, rare=False):
    """adversarial records with nothing due at once: no posted results, "Stopped" reported, no parse errors, no zones,
    every repeat timer armed and due 1 s to 30 years on; 5-field schedules on single minute / hour / day / month bits
    (`rare`: February 29th, 30th or 31st only)"""
    cols = population(rng, n, T, True)
    fl = cols["flags"]
    fl &= np.uint32(~(am.F_PENDING_OK | am.F_PENDING_FAIL | am.F_REMEDY_PENDING | am.F_REMEDY_OUTCOME_OK) & 0xFFFFFFFF)
    fl |= np.uint32(am.F_STOPPED_REPORTED | am.F_TIMER_ARMED)
    fl[:] = np.where((fl & 7) == am.KIND_PARSE_ERROR, (fl & ~np.uint32(7)) | am.KIND_STOPPED, fl)
    cols["finished_at"][:] = T - cols["ras"].astype(np.int64) + rng.integers(1, 30 * 366 * DAY, n)
    cr = (fl & 7) == am.KIND_CRON_SPEC
    m = int(cr.sum())
    bit = lambda lo, hi: np.uint64(1) << rng.integers(lo, hi, m).astype(np.uint64)
    cols["minute"][cr] = bit(0, 60)
    cols["hour"][cr] = bit(0, 24)
    star_dow = np.uint64((1 << 63) | 0x7F)
    if rare:
        cols["dom"][cr] = bit(29, 32)
        cols["month"][cr] = np.uint64(1 << 2)
        cols["dow"][cr] = star_dow
    else:
        cols["dom"][cr] = bit(1, 32)
        cols["month"][cr] = bit(1, 13)
        cols["dow"][cr] = np.where(rng.random(m) < 0.7, star_dow, bit(0, 7))
    return cols


ND_SIZES = [1, 2, 7, 64, 1000, 70_001]


@pytest.mark.parametrize("rare", [False, True], ids=["sparse", "rare"])
@pytest.mark.parametrize("T", INSTANTS, ids=_tid)
def test_next_due_far_ahead_equals_the_per_record_minimum(am, orc, T, rare):
    """am_sweep_next_due(T) on quiet populations of every size of ND_SIZES is exactly the per-record minimum: the
    device's Next() where it scans days to years ahead (Feb 29, the five-year give-up) and its grid-stride / shuffle /
    atomicMin reduction"""
    lib = orc.load()
    rng = np.random.default_rng(zlib.crc32(f"next due {T} {rare}".encode()))
    far = 0
    for n in ND_SIZES:
        cols = _quiet(am, rng, n, T, rare)
        want = _next_due_want(am, lib, cols, T)
        with am.Sweep(capacity=n) as s:
            s.load_range(0, cols)
            assert s.next_due(T) == want, (n, want)
        far += want is None or want - T > DAY
    assert far >= 2, far


HOLD_VARIANTS = ["hold", "hold_timeouts", "remedy_hold", "remedy_hold_timeouts"]


def _pair(am, zmap, cols, variant):
    """a handle with the variant's holds on and its model (a handle that never gets a non-zero wf_timeout sweeps with
    the hold-only variants, and the timeout oracle is then the hold oracle)"""
    return Pair(am, zmap, cols, hold=True, remedy=variant.startswith("remedy"))


def _busy(am, T, k, W):
    """a check due at T and every 5 s (or every minute), with a remedy and no runs limit: it is submitted and held"""
    rc, r = (am.classify(repeat_after_sec=5, finished_at=T - 100, has_remedy=True) if k % 2 == 0 else
             am.classify(cron="* * * * *", has_remedy=True))
    assert rc == 0
    r["wf_timeout"] = W
    return r


@pytest.mark.parametrize("T", [TS[0], 0, -1, 1 << 31, -(1 << 40), 1 << 54, LEAP_2000_END, END_2099], ids=_tid)
@pytest.mark.parametrize("variant", HOLD_VARIANTS)
def test_next_due_with_the_hold(am, orc, zmap, variant, T):
    """Quiet populations with a quarter of busy checks, submitted at T; half of those then get Failed (a remedy run
    starts for them under the remedy hold).  next_due at several seconds after the last tick, up to past every
    deadline, equals the per-record minimum on the oracle's state: a held record never wins by its schedule, a
    deadline D of either kind of run counts as max(D, T + 1)."""
    lib = orc.load()
    remedy, timeouts = variant.startswith("remedy"), variant.endswith("timeouts")
    rng = np.random.default_rng(zlib.crc32(f"next due hold {variant} {T}".encode()))
    hold_mattered = floor_mattered = remedy_deadlines = 0
    for n in (1, 64, 3000):
        cols = _quiet(am, rng, n, T)
        recs = am.columns_to_records(cols)
        busy = np.flatnonzero((np.arange(n) == 0) | (rng.random(n) < 0.25))
        for k, i in enumerate(busy):
            recs[i] = _busy(am, T, k, int(rng.integers(10, 100)) if timeouts else 0)[0]
        p = _pair(am, zmap, cols, variant)
        try:
            p.upsert(np.arange(n), recs)
            p.tick(T)
            assert p.m.in_flight()[0] == T
            failed = rng.choice(busy, (len(busy) + 1) // 2, replace=False)
            p.post(failed, np.full(len(failed), am.PHASE_FAILED, dtype=np.uint8))
            p.tick(T + 1)
            for dt in (1, 2, 9, 31, 101, 10 ** 6):
                t = T + 1 + dt
                runs = dict(since=p.m.since, deadline=p.m.deadline)
                if remedy:
                    runs.update(rsince=p.m.rsince, rdeadline=p.m.rdeadline)
                    remedy_deadlines += int(((p.m.rsince != NONE) & (p.m.rdeadline != NO_DEADLINE)).sum())
                want = _next_due_want(am, lib, p.m.cols(), t, **runs)
                assert p.s.next_due(t) == want, (n, t, want)
                hold_mattered += _next_due_want(am, lib, p.m.cols(), t) != want
                floor_mattered += _next_due_want(am, lib, p.m.cols(), t, floor=t, **runs) != want
        finally:
            p.close()
    assert hold_mattered > 0
    assert floor_mattered > 0 if timeouts else floor_mattered == 0
    assert remedy_deadlines > 0 if remedy and timeouts else remedy_deadlines == 0


def test_next_due_10m_records_one_winner(am, orc):
    """10 M armed interval checks due years ahead and, every seventh slot, the schedule that never fires: one record
    that wins alone — an interval check or a 5-field schedule — at slot 0, the last slot, 2^23 - 1 and the middle"""
    if _emulated(am):
        pytest.skip("10 M records: GPU only")
    lib = orc.load()
    n = 10_000_000
    T = TS[0]
    rng = np.random.default_rng(10)
    cols = am.alloc_columns(n)
    cron = np.arange(n) % 7 == 3
    cols["flags"][:] = np.where(cron, am.KIND_CRON_SPEC, am.KIND_INTERVAL).astype(np.uint32) | np.uint32(
        am.F_TIMER_ARMED | am.F_STOPPED_REPORTED)
    feb30 = am.cron_parse("0 0 30 2 *")
    for m in MASKS:
        cols[m][cron] = np.uint64(getattr(feb30, m))
    cols["ras"][:] = DAY
    cols["finished_at"][:] = T + 10 ** 8 + rng.integers(0, 10 ** 6, n)
    bulk = _next_due_want(am, lib, cols, T)
    assert bulk is not None and bulk > T + 10 ** 8
    every_day = am.cron_parse("17 3 * * *")
    with am.Sweep(capacity=n) as s:
        s.load_range(0, cols)
        assert s.next_due(T) == bulk
        for k, pos in enumerate([0, n - 1, (1 << 23) - 1, n // 2, 1 << 23]):
            one = {name: v[pos:pos + 1].copy() for name, v in cols.items()}
            if k % 2:
                one["flags"][:] = am.KIND_CRON_SPEC | am.F_STOPPED_REPORTED
                for m in MASKS:
                    one[m][:] = np.uint64(getattr(every_day, m))
            else:
                one["flags"][:] = am.KIND_INTERVAL | am.F_TIMER_ARMED | am.F_STOPPED_REPORTED
                one["finished_at"][:] = T - DAY + 777 + k
            want = _next_due_want(am, lib, one, T)
            assert T < want < bulk
            s.upsert([pos], am.columns_to_records(one))
            assert s.next_due(T) == want, (pos, want)
            s.upsert([pos], am.columns_to_records({name: v[pos:pos + 1] for name, v in cols.items()}))
        assert s.next_due(T) == bulk


# ---- 3. the hold sweep variants at the extreme instants ----------------------------------------------------------------
HOLD_SIZES = [1, 1023, 1025, 2500]
STEPS = test_remedy_hold_gpu.STEPS


@pytest.mark.parametrize("mode", [0, FULL, CATCH], ids=["plain", "full_scan", "catch_up"])
@pytest.mark.parametrize("T", TS, ids=_tid)
@pytest.mark.parametrize("variant", HOLD_VARIANTS)
def test_hold_variants_at_extreme_instants(am, zmap, variant, T, mode):
    """A random walk of upserts with wf_timeout, removes, loads, posts and the holds turned off and on between the
    ticks of STEPS from T, each tick compared with the oracle (list, statistics, columns, both in-flight reads and both
    timed-out lists).  Slot 0 keeps a check that is due every 5 s with a remedy and a workflow timeout of 1 s, so that
    every walk holds runs, times them out and starts remedy runs where the variant does."""
    remedy, timeouts = variant.startswith("remedy"), variant.endswith("timeouts")
    n = HOLD_SIZES[TS.index(T) % len(HOLD_SIZES)]
    rng = np.random.default_rng(zlib.crc32(f"hold variants {variant} {T} {mode}".encode()))
    tz = zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))

    def records(slots):
        recs = am.columns_to_records(population(rng, len(slots), T, True, tz))
        recs["wf_timeout"] = np.where(rng.random(len(slots)) < 0.2, 0, rng.integers(1, 120, len(slots))) if timeouts else 0
        recs[np.asarray(slots) == 0] = _busy(am, T, 0, 1 if timeouts else 0)
        return recs

    p = _pair(am, zmap, population(rng, n, T, True, tz), variant)
    held = timed = rtimed = 0
    try:
        p.upsert(np.arange(n), records(np.arange(n)))
        for k, step in enumerate(STEPS):
            if k:
                r = rng.random()
                if r < 0.25:
                    sl = rng.choice(n, min(n, 60), replace=False)
                    p.upsert(sl, records(sl))
                elif r < 0.33 and n > 1:
                    p.remove(rng.choice(np.arange(1, n), min(n - 1, 30), replace=False))
                elif r < 0.41 and n > 1:
                    m = min(200, n - 1)
                    p.load(int(rng.integers(1, n - m + 1)), population(rng, m, T, True, tz))
                elif r < 0.47:
                    p.set_hold(False)
                    p.set_hold(True)
                    if remedy:
                        p.set_remedy(True)
                busy = p.m.since != NONE
                if remedy:
                    busy |= p.m.rsince != NONE
                busy = np.flatnonzero(busy)
                if len(busy) and k % 2:
                    sl = rng.choice(busy, min(len(busy), 30), replace=False)
                    ph = np.where(rng.random(len(sl)) < 0.6, 2, rng.integers(0, 3, len(sl))).astype(np.uint8)
                    rp = np.where(rng.random(len(sl)) < 0.5, 0, rng.integers(1, 3, len(sl))).astype(np.uint8)
                    p.post(sl, ph, rp)
            T += step
            held += int((p.m.in_flight() != NONE).sum())
            out = p.tick(T, mode)
            timed += len(out[3][0])
            if remedy:
                rtimed += len(out[4][0])
        assert held > 0
        assert timed > 0 if timeouts else timed == 0
        if remedy:
            assert p.started > 0
            assert rtimed > 0 if timeouts else rtimed == 0
    finally:
        p.close()
