"""Change details (am_sweep_set_change_details / am_sweep_last_change_details): after every tick the handle's details
must equal the change-details oracle's (tests/change_details_oracle.py, in tests/handle_model.py), entry by
entry with the changed set.  Through every tick entry point: the hand-derived cases, the sparse and the dense result
routes with reads between posts and ticks, the hold, the hold with timeouts and the remedy hold, catch-up ticks on named
zones with AM_SWEEP_FULL_SCAN, closed loop, short buffers and refused ticks, the call contract, run_ticks, toggling
details and tracking, random call sequences through tests/test_call_sequences_gpu.py's walk, launch counts and 10 M
records."""
import zlib

import numpy as np
import pytest

import amgen
import change_details_cases
import change_details_oracle as cdo
import changes_oracle
from adversarial import ZoneMap, population, zones_usable
from handle_pair import check_details, emulated
from test_call_sequences_gpu import WALKS
from test_status_changes_gpu import CATCH, CLOSED, ENTRIES, FULL, ChangesWalk, pair
from timeout_cases import M0, rec

pytestmark = pytest.mark.gpu

DAY = 86400


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


# ---- 1. the hand-derived cases, through every tick entry point -------------------------------------------------------
@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("case", change_details_cases.CASES, ids=lambda c: c.__name__)
def test_hand_derived_cases(am, zmap, case, entry):
    p = pair(am, zmap, case.n, case.hold, entry=entry, details=True)
    try:
        case(am, p)
    finally:
        p.close()


# ---- 2. random walks: sparse and dense posts, reads in between, the holds and timeouts, every entry point ---------------
STEPS = [1, 1, 59, 1, 60, 2, 1, -60, 0, 1, 17, 1, 59, 1, 600, 1, 43, 1, -1, 120, 1, 30, 29, 1, 3617, 1, 5, 55, 1]


def _walk(am, zmap, hold, early, mode, seed_text, monkeypatch, n=3000):
    rng = np.random.default_rng(zlib.crc32(seed_text.encode()))
    T = M0 + 12 * DAY + 14 * 3600 - 3
    tz = zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))

    def records(k):
        r = am.columns_to_records(population(rng, k, T, True, tz))
        if hold == "remedy":
            r["wf_timeout"] = np.where(rng.random(k) < 0.2, 0, rng.integers(1, 120, k))
        return r

    monkeypatch.setenv("AMSWEEP_EARLY_RESULTS", str(early))
    p = pair(am, zmap, n, hold, details=True)
    try:
        p.upsert(np.arange(n), records(n))
        entries = ENTRIES + ["tick_short"]
        for k, step in enumerate(STEPS):
            if k:
                r = rng.random()
                if r < 0.2:
                    p.upsert(rng.choice(n, 60, replace=False), records(60))
                elif r < 0.28:
                    p.remove(rng.choice(n, 30, replace=False))
                elif r < 0.36:
                    first = int(rng.integers(0, n - 200))
                    p.load(first, am.records_to_columns(records(200)))
                dense = k % 4 == 3  # more than an eighth of the records: the sweep applies them
                sl = rng.choice(n, 1500 if dense else 40, replace=False)
                sl[-1] = sl[0]  # (two entries of one call)
                ph = rng.integers(0, 3, len(sl)).astype(np.uint8)
                rp = np.where(rng.random(len(sl)) < 0.5, 0, rng.integers(1, 3, len(sl))).astype(np.uint8)
                p.post(sl, ph, rp)
                if k % 3 == 1:  # a read between the post and the tick leaves the results pending
                    p.read(rng.choice(n, 10, replace=False))
                    if rng.random() < 0.5:
                        p.post(sl[:20], np.full(20, 1, np.uint8))
                if k % 7 == 5:  # details off for a tick, then on again
                    p.set_details(False)
                    T += step
                    p.tick(T, mode, entry=entries[k % len(entries)])
                    p.post(sl[20:30], np.full(10, 2, np.uint8))
                    p.set_details(True)
                    continue
            T += step
            p.tick(T, mode, entry=entries[k % len(entries)])
        return p.detailed
    finally:
        p.close()


@pytest.mark.parametrize("early", [1, 0], ids=["early_results", "in_sweep"])
@pytest.mark.parametrize("hold", [None, "hold", "remedy"])
@pytest.mark.parametrize("mode", [0, CATCH | FULL], ids=["plain", "catch_up_full"])
def test_random_walks_equal_the_oracle(am, zmap, hold, early, mode, monkeypatch):
    detailed = _walk(am, zmap, hold, early, mode, f"details {hold} {early} {mode}", monkeypatch)
    assert detailed > 1000, detailed


def test_closed_loop(am, zmap):
    n = 4000
    rng = np.random.default_rng(7)
    T = M0 + 3
    p = pair(am, zmap, n, details=True)
    try:
        p.upsert(np.arange(n), am.columns_to_records(population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY)))))
        for k, step in enumerate([0, 1, 57, 60, 1, 3600]):
            T += step
            if k % 2:
                sl = rng.choice(n, 300, replace=False)
                p.post(sl, rng.integers(0, 3, 300).astype(np.uint8), rng.integers(0, 3, 300).astype(np.uint8))
            p.tick(T, CLOSED | (FULL if k == 2 else 0) | (CATCH if k == 4 else 0), entry=ENTRIES[k % 4])
        assert p.detailed > 500, p.detailed
    finally:
        p.close()


# ---- 3. catch-up ticks on named zones (amgen config 22), the remedy hold with timeouts -----------------------------------
def test_catch_up_on_named_zones(am, zmap):
    n = 20_000
    T = amgen.T0_MON_0915
    cols = amgen.fill(22, 2, 0, n, T, am.load().am_healthcheck_classify)
    rng = np.random.default_rng(23)
    cols["flags"] |= np.where(rng.random(n) < 0.5, am.F_HAS_REMEDY, 0).astype(np.uint32)
    p = pair(am, zmap, n, "remedy", details=True)
    try:
        recs = am.columns_to_records(cols)
        recs["wf_timeout"] = rng.integers(0, 400, n)
        p.upsert(np.arange(n), recs)
        for k, step in enumerate([0, 60, 1, 150, 59, 600, 1, 3600, 61, 240]):
            T += step
            if k:
                sl = rng.choice(n, 1500, replace=False)
                p.post(sl, np.where(rng.random(1500) < 0.7, 2, 0).astype(np.uint8),
                       np.where(rng.random(1500) < 0.3, 1, 0).astype(np.uint8))
            p.tick(T, CATCH | (FULL if k % 3 == 0 else 0), entry=ENTRIES[k % 4])
        assert p.detailed > 5000, p.detailed
        det = p.m.details()
        assert (det["started"] != cdo.NONE).any()
    finally:
        p.close()


# ---- 4. the call contract ----------------------------------------------------------------------------------------------
def test_contract(am):
    """the switch, offset / cap / AM_E_NOSPACE / AM_E_RANGE, refused and AM_E_NOSPACE ticks, run_ticks"""
    import ctypes as C
    n = 64
    with am.Sweep(capacity=n, shard_base=1000) as s:
        lib = s._lib
        cnt = am.abi.u64(0)
        assert lib.am_sweep_set_change_details(s._h, 1) == am.AM_E_INVAL  # tracking off
        assert lib.am_sweep_last_change_details(s._h, 0, None, None, 0, C.byref(cnt)) == am.AM_E_INVAL
        s.set_track_changes(True)
        assert lib.am_sweep_last_change_details(s._h, 0, None, None, 0, C.byref(cnt)) == am.AM_E_INVAL  # details off
        s.set_change_details(True)
        assert len(s.last_change_details()[0]) == 0
        s.set_hold_in_flight(True)
        s.upsert(np.arange(10), np.concatenate([rec(am, 0, repeat_after_sec=60, finished_at=M0 - 100)] * 10))
        s.tick(M0)
        s.upsert([10], rec(am, 0, repeat_after_sec=0))
        s.post_result(np.arange(10), np.full(10, 1, np.uint8))
        with pytest.raises(am.AmError) as e:  # (slot 10 is reported STOPPED)
            s.tick(M0 + 1, cap=0)
        assert e.value.code == am.AM_E_NOSPACE
        idx, det = s.last_change_details()
        assert idx.tolist() == list(range(1000, 1011)) == s.last_changes()[0].tolist()
        assert det["started"].tolist() == [M0] * 10 + [int(cdo.NONE)]
        assert det["applied"].tolist() == [am.CHG_SUCCEEDED] * 10 + [am.CHG_STOPPED]
        assert det["action"].tolist() == [0] * 10 + [am.ACT_STOPPED]
        idx, det = s.last_change_details(offset=7)
        assert idx.tolist() == [1007, 1008, 1009, 1010]
        out_i = np.zeros(4, np.uint64)
        out_d = np.zeros(4, am.CHANGE_DETAIL)
        assert lib.am_sweep_last_change_details(s._h, 3, out_i.ctypes.data, out_d.ctypes.data, 4, C.byref(cnt)) == am.AM_E_NOSPACE
        assert cnt.value == 8 and out_i.tolist() == [1003, 1004, 1005, 1006] and (out_d["started"] == M0).all()
        assert lib.am_sweep_last_change_details(s._h, 3, out_i.ctypes.data, None, 4, C.byref(cnt)) == am.AM_E_INVAL
        assert lib.am_sweep_last_change_details(s._h, 11, None, None, 0, C.byref(cnt)) == am.AM_OK and cnt.value == 0
        assert lib.am_sweep_last_change_details(s._h, 12, None, None, 0, C.byref(cnt)) == am.AM_E_RANGE
        with pytest.raises(am.AmError):  # a refused tick leaves the list in place
            s.tick(M0 + 2 * DAY, mode=CATCH)
        assert len(s.last_change_details()[0]) == 11
        # run_ticks empties the list (it is refused while the hold is on)
        s.set_hold_in_flight(False)
        s.post_result([5], [1])
        s.run_ticks(M0 + 2, 3)
        assert len(s.last_change_details()[0]) == 0
        # tracking off turns details off
        s.set_track_changes(False)
        s.set_track_changes(True)
        assert lib.am_sweep_last_change_details(s._h, 0, None, None, 0, C.byref(cnt)) == am.AM_E_INVAL


# ---- 5. random call sequences through the sequence model ------------------------------------------------------------------
@pytest.mark.parametrize("k", [0, 2, 3, 5], ids=[WALKS[k][3] for k in (0, 2, 3, 5)])
def test_random_call_sequences(am, zmap, k):
    cap, base, T0, name = WALKS[k]
    walk = ChangesWalk(am, zmap, name, zlib.crc32(f"details {name}".encode()), cap, base, T0, details=True)
    walk.run()
    assert walk.checked > 20


# ---- 6. launch counts ----------------------------------------------------------------------------------------------------
def test_launch_counts(am):
    """a handle with details off launches what a tracking-only handle launches, also after on -> off"""
    n = 3000
    recs = np.concatenate([rec(am, 0, repeat_after_sec=60, finished_at=M0 - 100, has_remedy=True)] * n)
    with am.Sweep(capacity=n) as a, am.Sweep(capacity=n) as b, am.Sweep(capacity=n) as c:
        for s in (a, b, c):
            s.set_track_changes(True)
        b.set_change_details(True)
        b.set_change_details(False)
        counts = {id(s): [] for s in (a, b, c)}
        for k, t in enumerate([M0, M0 + 1, M0 + 30, M0 + 60, M0 + 61]):
            if k == 0:
                for s in (a, b, c):
                    s.upsert(np.arange(n), recs)
            if k == 3:
                c.set_change_details(True)
            sl = np.arange(0, n, 7 if k % 2 else 2)  # sparse and dense posts
            for s in (a, b, c):
                l0 = s.launch_count
                s.post_result(sl, np.full(len(sl), 2, np.uint8))
                s.read([1])
                s.tick(t)
                counts[id(s)].append(s.launch_count - l0)
        assert counts[id(a)] == counts[id(b)], counts
        # on: the read drain's two capture passes, the sweep's before the exceptions and the snapshot after the list
        assert [x - y for x, y in zip(counts[id(c)], counts[id(a)])][3:] == [4, 4], counts


# ---- 7. one check through its phases ---------------------------------------------------------------------------------------
def test_one_check_through_its_phases(am, zmap):
    """one check through Succeeded, Failed with a remedy, a remedy timeout and a reset: what a status write needs for
    each phase hcc.go:636-851 applies (StartedAt / RemedyStartedAt = then, the reset) is in the details alone"""
    p = pair(am, zmap, 4, "remedy", details=True)
    try:
        p.upsert([0], rec(am, 40, repeat_after_sec=60, finished_at=M0 - 100, has_remedy=True, remedy_runs_limit=5,
                          remedy_reset_interval=100000))
        T = M0
        p.tick(T)  # submitted at M0
        p.post([0], [1])
        p.tick(T + 5)
        (d,) = p.m.details()
        assert (d["started"], d["applied"]) == (M0, cdo.CHG_SUCCEEDED)  # Succeeded: StartedAt = then, FinishedAt = now
        p.tick(T + 65)  # submitted again
        p.post([0], [2])
        p.tick(T + 70)  # Failed: LastFailedAt = now, the remedy run starts
        (d,) = p.m.details()
        assert (d["started"], d["applied"]) == (T + 65, cdo.CHG_FAILED) and d["action"] & 0x02
        p.tick(T + 110)  # the remedy run outlives W = 40: RemedyFailed, RemedyStartedAt = then
        (d,) = p.m.details()
        assert (d["remedy_started"], d["applied"]) == (T + 70, cdo.CHG_REMEDY_FAILED | cdo.CHG_REMEDY_TIMED_OUT)
        p.tick(T + 200)  # submitted again
        p.post([0], [1])
        p.tick(T + 205)  # Succeeded with RemedyTotalRuns >= 1: "HealthCheck Passed so Remedy is reset"
        (d,) = p.m.details()
        assert d["action"] & 0x20 and d["applied"] == cdo.CHG_SUCCEEDED and d["started"] == T + 200
    finally:
        p.close()


# ---- 8. full size, on the GPU only -----------------------------------------------------------------------------------------
def test_full_size_config3(am, zmap):
    """one 10 M-record config 3 tick (the dense route), the details compared in full"""
    if emulated(am):
        pytest.skip("10 M records: GPU only")
    n = 10_000_000
    T0 = amgen.T0_MON_0915
    cols = amgen.fill(3, 3, 0, n, T0, am.load().am_healthcheck_classify)
    with am.Sweep(capacity=n) as s:
        s.set_track_changes(True)
        s.set_change_details(True)
        s.load_range(0, cols)
        before = changes_oracle.snapshot(cols)
        out = zmap.sweep(cols, T0)
        want = changes_oracle.changed(before, cols, out[0], out[1])
        s.tick_view(T0)
        assert len(want) > 7_000_000, len(want)
        check_details(s, want, cdo.details(want, before["flags"], out, T0, 0, {}, {}), "config 3")
