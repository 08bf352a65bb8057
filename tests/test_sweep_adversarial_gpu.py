"""The adversarial population (tests/adversarial.py) on the device, through the C-ABI, against the C oracle
applied tick by tick: single ticks of every kernel variant at ragged sizes, runs of ticks (blocked at
several block lengths and unblocked, open and closed loop, across zones whose UTC offset is a half hour
or has seconds), am_sweep_next_due against a brute-force search, and records bound to zone ids that the
process never registered."""
import numpy as np
import pytest

from adversarial import (TS, ZoneMap, first_difference, population, run_single_ticks, zones_usable)

pytestmark = pytest.mark.gpu

T0 = 1789982100          # 2026-09-21 09:15:00 UTC Monday
T_MONROVIA = 44618405    # 1971-06-01 10:00:05 UTC: Monrovia's clock reads 09:15:35 (UTC-0:44:30)


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


SIZES = [1, 1023, 1025, 2500, 70_001]


@pytest.mark.parametrize("in_domain", [True, False], ids=["library-domain", "beyond-domain"])
@pytest.mark.parametrize("seed", range(12))
def test_adversarial_single_ticks(am, zmap, seed, in_domain):
    """Three consecutive host ticks, all four kernel variants (open / closed loop x with / without the
    cron masks), at every instant of TS: list, action bytes, statistics and all sixteen columns."""
    n = SIZES[seed % len(SIZES)]
    for mode in (0, am.SWEEP_CLOSED_LOOP, am.SWEEP_FULL_SCAN, am.SWEEP_CLOSED_LOOP | am.SWEEP_FULL_SCAN):
        bad = run_single_ticks(am.Sweep, zmap, seed, n, TS[seed % len(TS)], mode, in_domain)
        assert bad is None, bad


def _stats_rows(am, stats, k):
    return {f: int(stats[f][k]) for f in am.abi.STAT_FIELDS}


RUNS = [  # id, first tick (off the minute), ticks, library domain
    ("2026", T0 + 17, 300, True),            # every generator zone: Lord Howe +10:30, Kathmandu +5:45, St John's -2:30
    ("1971-monrovia", T_MONROVIA, 200, True),  # and Monrovia -0:44:30: the local minute starts at UTC second 30
    ("epoch", 23, 150, True),
    ("2038", (1 << 31) + 7, 257, True),
    ("-2^40", -(1 << 40) + 31, 180, True),
    ("2^54", (1 << 54) + 13, 150, True),
    ("beyond-2026", T0 + 41, 220, False),
    ("beyond--2^33", -(1 << 33) + 5, 160, False),
]


@pytest.mark.parametrize("closed", [False, True], ids=["open", "closed"])
@pytest.mark.parametrize("run_id,T,nt,in_domain", RUNS, ids=[r[0] for r in RUNS])
def test_adversarial_run_of_ticks_blocked_and_unblocked(am, zmap, monkeypatch, run_id, T, nt, in_domain, closed):
    """am_sweep_run_ticks unblocked and with AM_SWEEP_BLOCKED at block lengths 1, 7, 96 and 128: every
    blocked run equals the unblocked one (per-tick statistics and the columns afterwards); in the library's
    domain both equal the oracle tick by tick."""
    n, seed = 3000, 1000 + RUNS.index((run_id, T, nt, in_domain))
    rng = np.random.default_rng(seed)
    cols = population(rng, n, T, in_domain, zmap.ids_of(zones_usable(T, T + nt)))
    mode = am.SWEEP_CLOSED_LOOP if closed else 0
    runs = {}
    for block in (0, 1, 7, 96, 128):
        if block:
            monkeypatch.setenv("AMSWEEP_BLOCK_TICKS", str(block))
        with am.Sweep(capacity=n) as s:
            s.load_range(0, cols)
            stats = s.run_ticks(T, nt, mode=mode | (am.SWEEP_BLOCKED if block else 0), seed=seed)
            runs[block] = (stats, s.read_range(0, n))
    plain, plain_cols = runs[0]
    for block in (1, 7, 96, 128):
        stats, dev = runs[block]
        for k in range(nt):
            assert _stats_rows(am, stats, k) == _stats_rows(am, plain, k), f"block {block} tick {k}"
        for name in am.COLUMN_NAMES:
            np.testing.assert_array_equal(dev[name], plain_cols[name], err_msg=f"block {block}: {name}")
    if not in_domain:
        return
    ocols = {k: v.copy() for k, v in cols.items()}
    emitted = 0
    for k in range(nt):
        _, _, ws = zmap.sweep(ocols, T + k, mode=mode, seed=seed)
        assert _stats_rows(am, plain, k) == ws, f"tick {k}"
        emitted += ws["n_emitted"]
    assert emitted > nt
    for name in am.COLUMN_NAMES:
        np.testing.assert_array_equal(plain_cols[name], ocols[name], err_msg=name)


def _first_active_tick(zmap, cols, T, horizon):
    """The first t in (T, T + horizon] at which the oracle's open-loop tick emits something or changes a
    column (a posted result applied without an action), or None."""
    o = {k: v.copy() for k, v in cols.items()}
    ref = b"".join(v.tobytes() for v in o.values())
    for t in range(T + 1, T + horizon + 1):
        idx, _, _ = zmap.sweep(o, t)
        if len(idx) or b"".join(v.tobytes() for v in o.values()) != ref:
            return t
    return None


NEXT_DUE_T = [T0 + 17, T0, T0 + 59, 1790812799, T_MONROVIA, T_MONROVIA - 5, 31535999, 17, 1709164799]


@pytest.mark.parametrize("zones", [False, True], ids=["utc", "zone-bound"])
def test_next_due_by_brute_force(am, zmap, zones):
    """am_sweep_next_due(T) on small populations (1..64 records) from the adversarial generator: without
    zone-bound records it is exactly the first second in (T, T + H] at which a tick does anything; with them
    it may be earlier, never later, and never <= T.  Either way the library's own ticks strictly between T and
    it emit nothing."""
    H = 1900
    every_minute = am.cron_parse("* * * * *")
    rng = np.random.default_rng(77 if zones else 76)
    cases = 0
    for case in range(72):
        T = NEXT_DUE_T[(case // 4) % len(NEXT_DUE_T)]
        n = int(min(64, rng.geometric(0.2)))
        tz_ids = zmap.ids_of(zones_usable(T, T + H)) if zones else []
        cols = population(rng, n, T, True, tz_ids)
        fl = cols["flags"]
        if case % 4:  # quiet: no posted results, "Stopped" reported, no parse errors
            fl &= ~np.uint32(am.F_PENDING_OK | am.F_PENDING_FAIL | am.F_REMEDY_PENDING | am.F_REMEDY_OUTCOME_OK)
            fl |= np.uint32(am.F_STOPPED_REPORTED)
            fl[:] = np.where((fl & 7) == am.KIND_PARSE_ERROR, (fl & ~np.uint32(7)) | am.KIND_STOPPED, fl)
        if case % 4 == 2:  # ... and every repeat timer armed
            fl |= np.uint32(am.F_TIMER_ARMED)
        if case % 4 == 3:  # 5-field schedules only, every fourth of them "* * * * *" (in one of the zones)
            fl[:] = (fl & ~np.uint32(7)) | am.KIND_CRON_SPEC
            star = rng.integers(0, 4, n) == 0
            for name in ("minute", "hour", "dom", "month", "dow"):
                cols[name][star] = np.uint64(getattr(every_minute, name))
            if tz_ids:
                zone = np.array(tz_ids, dtype=np.uint32)[rng.integers(0, len(tz_ids), n)]
                fl[star] = (fl[star] & np.uint32(0x00FFFFFF)) | (zone[star] << np.uint32(24))
        bound = ((fl & 7) == am.KIND_CRON_SPEC) & ((fl >> 24) != 0) & ((fl & am.F_TOMBSTONE) == 0)
        assert zones or not bound.any()
        want = _first_active_tick(zmap, cols, T, H)
        with am.Sweep(capacity=n) as s:
            s.load_range(0, cols)
            nd = s.next_due(T)
            if bound.any():
                assert nd is not None and nd > T, (case, T, nd)
                assert want is None or nd <= want, (case, T, nd, want)
            elif want is None:
                assert nd is None or nd > T + H, (case, T, nd)
            else:
                assert nd == want, (case, T, nd, want)
            quiet = min(nd if nd is not None else T + H + 1, T + 241) - 1 - T  # (at most four minutes of them)
            if quiet > 0:
                stats = s.run_ticks(T + 1, quiet)
                assert int(stats["n_emitted"].sum()) == 0, (case, T, nd)
        cases += want is not None and (want - T) > 1
    assert cases >= 8  # the populations do not all act at once
    if zones:  # in a zone whose offset has seconds the local minute starts mid-way through the UTC one
        rc, r = am.classify(cron="CRON_TZ=Africa/Monrovia * * * * *", finished_at=T_MONROVIA - 5)
        assert rc == 0
        cols = am.records_to_columns(r)
        want = _first_active_tick(zmap, cols, T_MONROVIA, 120)
        assert want == T_MONROVIA + 25  # 10:00:30 UTC = 09:16:00 in Monrovia
        with am.Sweep(capacity=1) as s:
            s.load_range(0, cols)
            nd = s.next_due(T_MONROVIA)
            assert T_MONROVIA < nd <= want, nd
            assert len(s.tick(want)[0]) == 1


def test_zone_ids_outside_the_registry_are_rejected(am, zmap):
    """Flags bits 24..31 name a zone of this process's registry.  A CRON_SPEC record with an id nobody
    registered (a snapshot from another process, say) is refused by am_sweep_load_range and am_sweep_upsert
    with AM_E_INVAL and nothing of the call takes effect; the valid zone-bound records next to it are
    evaluated as before."""
    bad_id = 200  # far above the zones of this test process
    specs = ["CRON_TZ=Asia/Kathmandu * * * * *", "CRON_TZ=Australia/Lord_Howe */2 * * * *", "*/3 * * * *",
             "CRON_TZ=Africa/Monrovia * * * * *"]
    recs = np.concatenate([am.classify(cron=sp, finished_at=T0 - 5)[1] for sp in specs])
    assert all(recs["flags"][:2] >> 24 != 0) and recs["flags"][3] >> 24 == zmap.ids["Africa/Monrovia"]
    bad = recs[:1].copy()
    bad["flags"] = (bad["flags"] & 0x00FFFFFF) | (bad_id << 24)
    n = 8
    with am.Sweep(capacity=n) as s:
        s.load_range(0, am.records_to_columns(recs))
        before = s.read_range(0, n)
        mixed = am.records_to_columns(np.concatenate([recs[:2], bad, recs[2:]]))
        with pytest.raises(am.AmError) as e:
            s.load_range(0, mixed)
        assert e.value.code == am.AM_E_INVAL
        with pytest.raises(am.AmError) as e:
            s.upsert([4, 5], np.concatenate([recs[1:2], bad]))
        assert e.value.code == am.AM_E_INVAL
        after = s.read_range(0, n)
        for name in am.COLUMN_NAMES:
            np.testing.assert_array_equal(after[name], before[name], err_msg=name)
        assert s.size == len(recs)
        # a tick and a run of ticks see exactly the valid records, in 2026 and in Monrovia's 1971
        ocols = s.read_range(0, len(recs))
        for T in (T0, T0 + 60, T0 + 120, T0 + 121, 44618430, 44618490):
            gi, ga, gs = s.tick(T)
            wi, wa, ws = zmap.sweep(ocols, T)
            assert first_difference(am, (gi, ga, gs), (wi, wa, ws), s.read_range(0, len(recs)), ocols) is None, T
        for blocked in (0, am.SWEEP_BLOCKED):
            for start in (T0 - 7, 44618405):
                stats = s.run_ticks(start, 130, mode=blocked)
                for k in range(130):
                    _, _, ws = zmap.sweep(ocols, start + k)
                    assert _stats_rows(am, stats, k) == ws, (blocked, start, k)
