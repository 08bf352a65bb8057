"""Catch-up ticks (AM_SWEEP_CATCH_UP): a 5-field schedule is due iff it fires at some second of (P, T], P the
handle's previous tick; everything else happens once, at T.  Compared with the brute-force window oracle
(tests/window_oracle.py), with plain ticks of a second handle, and with the union of the plain ticks at
P+1 .. T."""
import calendar

import numpy as np
import pytest

import oracle_c
import window_oracle
from adversarial import MONROVIA, ZoneMap, first_difference, population, zones_usable

pytestmark = pytest.mark.gpu

DAY, HOUR = 86400, 3600
T_OCT = 1790812800  # 2026-10-01 00:00:00 UTC, Thursday
MODES = [0, 1, 2, 3]  # closed loop x FULL_SCAN


def utc(*a):
    return calendar.timegm(a + (0,) * (6 - len(a)))


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def _post_results(am, s, ocols, n, dense, seed):
    """workflow and remedy phases posted on every 2nd (dense) or 23rd (sparse) slot; the oracle's columns get
    the same pending bits"""
    rng = np.random.default_rng(seed)
    slots = np.arange(int(rng.integers(0, 23)), n, 2 if dense else 23)
    phase = rng.integers(1, 3, len(slots)).astype(np.uint8)
    rphase = rng.integers(0, 3, len(slots)).astype(np.uint8)
    s.post_result(slots, phase)
    s.post_result(slots, np.zeros_like(phase), rphase)
    hc = np.uint32(am.F_PENDING_OK | am.F_PENDING_FAIL)
    rm = np.uint32(am.F_REMEDY_PENDING | am.F_REMEDY_OUTCOME_OK)
    f = ocols["flags"][slots]
    f = (f & ~hc) | np.where(phase == am.PHASE_SUCCEEDED, am.F_PENDING_OK, am.F_PENDING_FAIL).astype(np.uint32)
    rbits = np.where(rphase == am.PHASE_SUCCEEDED, rm, np.uint32(am.F_REMEDY_PENDING)).astype(np.uint32)
    ocols["flags"][slots] = np.where(rphase != 0, (f & ~rm) | rbits, f)
    return slots


def _check(am, s, got, want, ocols, what):
    bad = first_difference(am, got, want, s.read_range(0, len(ocols["flags"])), ocols)
    assert bad is None, (what, bad)


def _same(am, a, b, n, what):
    """two handles' ticks (list, statistics, every column) equal byte for byte"""
    (ai, aa, ast), (bi, ba, bst) = a, b
    assert ast == bst, what
    np.testing.assert_array_equal(ai, bi, err_msg=str(what))
    np.testing.assert_array_equal(aa, ba, err_msg=str(what))


# ---- 1. a window with T's minute start as its only one (or none) is a plain tick ------------------------------
@pytest.mark.parametrize("n", [1, 1000, 70_001])
@pytest.mark.parametrize("mode", MODES)
def test_catch_up_with_one_or_no_minute_start_is_the_plain_tick(am, zmap, n, mode):
    rng = np.random.default_rng(1000 + n + mode)
    for T in [T_OCT + 13 * DAY + 14 * HOUR, 1789982100, 1789982100 + 30, T_OCT + 5 * HOUR + 60 * 7 + 45]:
        # (P, T] = (T - 59, T] holds exactly T's minute start when T is on the minute; (T - 20, T] off it holds none
        P = T - 59 if T % 60 == 0 else T - 20
        cols = population(rng, n, P, True, zmap.ids_of(zones_usable(P, T)))
        ocols = {k: v.copy() for k, v in cols.items()}
        with am.Sweep(capacity=n) as a, am.Sweep(capacity=n) as b:
            for s in (a, b):
                s.load_range(0, cols)
                s.set_seed(7)
            want = zmap.sweep(ocols, P, mode=mode & 1, seed=7)
            _check(am, a, a.tick(P, mode=mode), want, ocols, (n, mode, P))
            b.tick(P, mode=mode)
            got = a.tick(T, mode=mode | am.SWEEP_CATCH_UP)
            plain = b.tick(T, mode=mode)
            _same(am, got, plain, n, (n, mode, T))
            # T the only minute start of the window, in every zone: the catch-up tick IS the plain tick (the
            # on-minute one reads the planes and, with zones registered, launches tz_words_kernel: same kernels)
            assert a.launch_count == b.launch_count, (n, mode, T)
            want = zmap.sweep(ocols, T, mode=mode & 1, seed=7)
            _check(am, a, got, want, ocols, (n, mode, T))
            for name in am.COLUMN_NAMES:
                np.testing.assert_array_equal(a.read_range(0, n)[name], b.read_range(0, n)[name], err_msg=name)


# ---- 2. windows of every length from awkward start points, against the window oracle --------------------------
LENGTHS = [2, 59, 60, 61, 3599, 3600, 3601, 86399, 86400]
STARTS = {
    "on-minute": T_OCT + 12 * DAY + 14 * HOUR,
    "off-minute": T_OCT + 12 * DAY + 14 * HOUR + 17,
    "before-midnight": T_OCT + 20 * DAY - 1,
    "end-of-month": utc(2026, 10, 31, 23, 59, 30),
    "leap-february": utc(2028, 2, 28, 23, 59, 45),
    "new-year": utc(2026, 12, 31, 23, 59, 50),
}


@pytest.mark.parametrize("start", list(STARTS))
@pytest.mark.parametrize("closed,dense", [(False, False), (False, True), (True, False), (True, True)])
def test_windows_equal_the_window_oracle(am, zmap, start, closed, dense):
    P0 = STARTS[start]
    n = 3000
    mode = am.SWEEP_CLOSED_LOOP if closed else 0
    rng = np.random.default_rng(hash((start, closed, dense)) & 0xFFFF)
    with am.Sweep(capacity=n) as s:
        s.set_seed(11)
        for L in LENGTHS:
            P, T = P0, P0 + L
            cols = population(rng, n, T, True, zmap.ids_of(zones_usable(P, T)))
            ocols = {k: v.copy() for k, v in cols.items()}
            s.load_range(0, cols)
            _check(am, s, s.tick(P, mode=mode), zmap.sweep(ocols, P, mode=mode, seed=11), ocols, (start, L, "P"))
            _post_results(am, s, ocols, n, dense, L)
            got = s.tick(T, mode=mode | am.SWEEP_CATCH_UP)
            want = window_oracle.sweep_window(zmap, ocols, P, T, mode=mode, seed=11)
            _check(am, s, got, want, ocols, (start, L))


# ---- 3. short windows: the union of the plain ticks at P+1 .. T, no oracle -------------------------------------
def _cron_only(am, rng, n, tz_ids):
    c = am.alloc_columns(n)
    for name, (lo, hi) in {"minute": (0, 59), "hour": (0, 23), "dom": (1, 31), "month": (1, 12), "dow": (0, 6)}.items():
        full = sum(1 << v for v in range(lo, hi + 1))
        v = rng.integers(0, 1 << 62, n, dtype=np.uint64) & np.uint64(full)
        v[rng.random(n) < 0.5] = np.uint64(full)
        one = rng.random(n) < 0.2
        v[one] = (np.uint64(1) << rng.integers(lo, hi + 1, n).astype(np.uint64))[one]
        v |= np.where(rng.random(n) < 0.3, np.uint64(1 << 63), np.uint64(0))
        c[name][:] = v
    flags = np.full(n, am.KIND_CRON_SPEC, dtype=np.uint32)
    if tz_ids:
        z = np.array([0] + list(tz_ids), dtype=np.uint32)[rng.integers(0, len(tz_ids) + 1, n)]
        flags |= z << np.uint32(24)
    c["flags"][:] = flags
    return c


@pytest.mark.parametrize("P,L", [(T_OCT + 3 * HOUR + 59, 2), (T_OCT + 3 * HOUR + 31, 59), (T_OCT + 3 * HOUR + 7, 61),
                                 (T_OCT + 23 * HOUR + 58 * 60 + 13, 191), (utc(1971, 3, 4, 23, 58, 20), 200)])
def test_catch_up_emits_the_union_of_the_plain_ticks(am, zmap, P, L):
    n = 4000
    rng = np.random.default_rng(P % 1000 + L)
    cols = _cron_only(am, rng, n, zmap.ids_of(zones_usable(P, P + L)))
    with am.Sweep(capacity=n) as a, am.Sweep(capacity=n) as b:
        a.load_range(0, cols)
        b.load_range(0, cols)
        a.tick(P)
        b.tick(P)
        union = set()
        for t in range(P + 1, P + L + 1):
            union |= set(b.tick(t)[0].tolist())
        got = a.tick(P + L, mode=am.SWEEP_CATCH_UP)[0].tolist()
        assert got == sorted(union)
        assert len(union) > n // 50


# ---- 4. coalescing and one-shot actions --------------------------------------------------------------------------
def test_actions_happen_once_at_T(am):
    T0 = T_OCT + 8 * HOUR
    P, T = T0, T0 + HOUR
    recs = [am.classify(cron="* * * * *", finished_at=P - 5),             # 0: fires 60 times in the window
            am.classify(repeat_after_sec=60, finished_at=P - 100),        # 1: interval, due
            am.classify(repeat_after_sec=7200, finished_at=P - 100),      # 2: interval, not due
            am.classify(cron="0 9 * * *"),                                # 3: 09:00 is T itself
            am.classify(cron="30 7 * * *"),                               # 4: 07:30 is before the window
            am.classify(repeat_after_sec=3600, finished_at=P - 100),      # 5: gets a posted result
            am.classify(cron="15 8 * * *")]                               # 6: posted result, fires at 08:15
    rec = np.concatenate([r[1] for r in recs])
    late = np.concatenate([am.classify(repeat_after_sec=0)[1], am.classify(cron="bad cron")[1]])  # 7: STOPPED, 8: PARSE_ERROR
    with am.Sweep(capacity=16) as s, am.Sweep(capacity=16) as b:
        for h in (s, b):
            h.upsert(np.arange(len(rec)), rec)
            h.tick(P)
            h.upsert([7, 8], late)  # staged during the stall
            h.post_result([5, 6], [am.PHASE_SUCCEEDED, am.PHASE_FAILED])
        idx, act, st = s.tick(T, mode=am.SWEEP_CATCH_UP)
        got = dict(zip(idx.tolist(), act.tolist()))
        assert got == {0: am.ACT_SUBMIT_HC, 1: am.ACT_SUBMIT_HC, 3: am.ACT_SUBMIT_HC, 6: am.ACT_SUBMIT_HC,
                       7: am.ACT_STOPPED, 8: am.ACT_PARSE_ERROR}, got
        assert st["n_result_ok"] == 1 and st["n_result_fail"] == 1 and st["n_emitted"] == 6
        dev = s.read_range(0, 9)
        assert dev["finished_at"][5] == T and dev["finished_at"][6] == T and dev["finished_at"][7] == T
        assert dev["success"][5] == 1 and dev["failed"][6] == 1
        # the interval checks, STOPPED and PARSE_ERROR exactly as a plain tick at T would emit them
        pi, pa, _ = b.tick(T)
        plain = dict(zip(pi.tolist(), pa.tolist()))
        for k in (1, 2, 5, 7, 8):
            assert got.get(k) == plain.get(k), k
        # a second catch-up tick one second later (no minute start): STOPPED is not repeated, PARSE_ERROR is
        # (once per call), the interval check stays due
        idx, act, _ = s.tick(T + 1, mode=am.SWEEP_CATCH_UP)
        assert dict(zip(idx.tolist(), act.tolist())) == {1: am.ACT_SUBMIT_HC, 8: am.ACT_PARSE_ERROR}


# ---- 5. zones: daylight-saving changes, half-hour and quarter-hour offsets, an offset with seconds ---------------
ZONE_WINDOWS = [  # (zone, P, T, spec whose local time is skipped / repeated in the window, "skipped" | "repeated")
    ("Europe/Paris", utc(2026, 3, 28, 23, 10, 7), utc(2026, 3, 29, 4, 0, 0), "30 2 29 3 *", "skipped"),
    ("Europe/Paris", utc(2026, 10, 24, 22, 59, 59), utc(2026, 10, 25, 3, 0, 1), "30 2 25 10 *", "repeated"),
    ("America/New_York", utc(2026, 3, 8, 5, 0, 0), utc(2026, 3, 8, 9, 0, 0), "30 2 8 3 *", "skipped"),
    ("America/New_York", utc(2026, 10, 31, 12, 0, 13), utc(2026, 11, 1, 12, 0, 12), "30 1 1 11 *", "repeated"),
    ("Australia/Lord_Howe", utc(2026, 10, 3, 12, 0, 0), utc(2026, 10, 3, 18, 0, 0), "15 2 4 10 *", "skipped"),
    ("Australia/Lord_Howe", utc(2026, 4, 4, 13, 0, 0), utc(2026, 4, 4, 17, 0, 0), "45 1 5 4 *", "repeated"),
    # the most boxes: a 30-minute offset change inside a day-long window with partial first and last hours
    ("Australia/Lord_Howe", utc(2026, 10, 3, 15, 30, 0) - 40000 + 13, utc(2026, 10, 3, 15, 30, 0) + 46413, "15 2 4 10 *",
     "skipped"),
    ("Asia/Kathmandu", utc(2026, 10, 1, 6, 10, 0), utc(2026, 10, 1, 6, 20, 0), "0 12 1 10 *", None),
    (MONROVIA, utc(1971, 6, 1, 11, 30, 0), utc(1971, 6, 1, 12, 0, 0), "0 11 1 6 *", None),
]


@pytest.mark.parametrize("case", ZONE_WINDOWS, ids=lambda c: "{}-{}-{}".format(c[0].split("/")[-1], c[1], c[4]))
def test_zone_windows(am, zmap, case):
    zone, P, T, spec, what = case
    n = 2000
    rng = np.random.default_rng(P % 9973)
    zid = zmap.ids[zone]
    cols = _cron_only(am, rng, n, [zid])
    rc, special = am.classify(cron=f"CRON_TZ={zone} {spec}")
    assert rc == 0 and special["flags"][0] >> 24 == zid
    for name in am.COLUMN_NAMES:
        cols[name][0] = special[name][0]
    ocols = {k: v.copy() for k, v in cols.items()}
    with am.Sweep(capacity=n) as s:
        s.load_range(0, cols)
        _check(am, s, s.tick(P), zmap.sweep(ocols, P), ocols, (zone, P))
        got = s.tick(T, mode=am.SWEEP_CATCH_UP)
        want = window_oracle.sweep_window(zmap, ocols, P, T)
        _check(am, s, got, want, ocols, (zone, T))
        emitted = got[0].tolist()
        if what == "skipped":
            assert 0 not in emitted
        else:
            assert emitted.count(0) == 1
        assert len(emitted) > n // 100


# ---- 6. edges ------------------------------------------------------------------------------------------------------
def _cron_pop(am, n, T):
    rng = np.random.default_rng(6)
    return _cron_only(am, rng, n, [])


def test_first_tick_and_backwards_ticks_are_plain(am):
    n, T = 500, T_OCT + 9 * HOUR
    cols = _cron_pop(am, n, T)
    with am.Sweep(capacity=n) as a, am.Sweep(capacity=n) as b:
        a.load_range(0, cols)
        b.load_range(0, cols)
        _same(am, a.tick(T, mode=am.SWEEP_CATCH_UP), b.tick(T), n, "first")
        _same(am, a.tick(T - 3600, mode=am.SWEEP_CATCH_UP), b.tick(T - 3600), n, "T < P")
        _same(am, a.tick(T - 3600, mode=am.SWEEP_CATCH_UP), b.tick(T - 3600), n, "T == P")


def test_a_window_longer_than_a_day_is_refused_without_effect(am, zmap):
    n, T = 300, T_OCT + 9 * HOUR + 30
    cols = _cron_pop(am, n, T)
    cols["flags"][:10] = am.KIND_INTERVAL
    cols["ras"][:10] = 60
    ocols = {k: v.copy() for k, v in cols.items()}
    with am.Sweep(capacity=n) as s:
        s.load_range(0, cols)
        _check(am, s, s.tick(T), oracle_c.sweep(ocols, T), ocols, "P")
        new = am.columns_to_records({k: v[:2].copy() for k, v in ocols.items()})
        new["minute"][:] = 1
        s.upsert([20, 21], new)
        for name in am.COLUMN_NAMES:
            ocols[name][20:22] = new[name]
        _post_results(am, s, ocols, n, False, 3)
        with pytest.raises(am.AmError) as e:
            s.tick(T + DAY + 1, mode=am.SWEEP_CATCH_UP)
        assert e.value.code == am.AM_E_RANGE
        # nothing was drained and P did not move: a catch-up tick at P + 86400 is accepted, sees the staged calls and
        # equals the window oracle over the original (P, P + 86400]
        got = s.tick(T + DAY, mode=am.SWEEP_CATCH_UP)
        _check(am, s, got, window_oracle.sweep_window(zmap, ocols, T, T + DAY), ocols, "after")
        assert got[2]["n_result_ok"] + got[2]["n_result_fail"] > 0
        _check(am, s, s.tick(T + DAY + 1), oracle_c.sweep(ocols, T + DAY + 1), ocols, "plain")


def test_run_ticks_refuses_the_bit(am):
    with am.Sweep(capacity=10) as s:
        with pytest.raises(am.AmError) as e:
            s.run_ticks(T_OCT, 5, mode=am.SWEEP_CATCH_UP)
        assert e.value.code == am.AM_E_INVAL


@pytest.mark.parametrize("entry", ["tick", "tick_view", "tick_device", "tick_shard", "run_ticks", "run_ticks_blocked"])
def test_every_entry_point_sets_the_previous_tick(am, entry):
    n, X = 300, T_OCT + 10 * HOUR + 7
    with am.Sweep(capacity=n) as s:
        s.load_range(0, _cron_pop(am, n, X))
        if entry == "tick":
            s.tick(X)
        elif entry == "tick_view":
            s.tick_view(X)
        elif entry == "tick_device":
            s.tick_device(X, 0, 0, 0, 0, 0)
        elif entry == "tick_shard":
            s.tick_shard(X)
        else:
            s.run_ticks(X - 9, 10, mode=am.SWEEP_BLOCKED if entry == "run_ticks_blocked" else 0)
        # P == X: X + 86401 is a day and a second away (refused), X + 86400 is not
        with pytest.raises(am.AmError) as e:
            s.tick(X + DAY + 1, mode=am.SWEEP_CATCH_UP)
        assert e.value.code == am.AM_E_RANGE
        s.tick(X + DAY, mode=am.SWEEP_CATCH_UP)
