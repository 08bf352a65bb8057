"""Status changes (am_sweep_set_track_changes / am_sweep_last_changes): after every tick the handle's changed set must
equal the changed-set oracle's (tests/changes_oracle.py, the column diff of the model's states, tests/handle_model.py),
and the columns it returns the model's columns of those slots.  Through every tick entry point: the hand-derived cases, the
sparse and the dense result routes with reads between posts and ticks, the hold with timeouts and the remedy hold,
catch-up ticks on named zones with AM_SWEEP_FULL_SCAN and closed loop, short buffers, refused ticks, the call contract,
run_ticks, the switch, random call sequences through tests/test_call_sequences_gpu.py's walk, launch counts and 10 M
records."""
import os
import zlib

import numpy as np
import pytest

import amgen
import changes_cases
import changes_oracle
from adversarial import ZoneMap, population, zones_usable
from handle_pair import Pair, check_changes, emulated
from test_call_sequences_gpu import WALKS, Walk
from timeout_cases import M0, rec

pytestmark = pytest.mark.gpu

DAY = 86400
CLOSED, FULL, CATCH = 0x1, 0x2, 0x8
ENTRIES = ["tick", "tick_view", "tick_device", "tick_shard"]
STATUS = ["flags", "finished_at", "success", "failed", "remedy_success", "remedy_failed", "remedy_total",
          "remedy_finished_at"]


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def pair(am, zmap, n, hold=None, **kw):
    """a handle with tracking on and its model.  hold: None (off), "hold" (the hold in flight) or "remedy" (the hold,
    workflow timeouts and the remedy hold)"""
    return Pair(am, zmap, n, hold=hold is not None, remedy=hold == "remedy", track=True, every_slot=False, **kw)


# ---- 1. the hand-derived cases, through every tick entry point -------------------------------------------------------
@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("case", changes_cases.CASES, ids=lambda c: c.__name__)
def test_hand_derived_cases(am, zmap, case, entry):
    p = pair(am, zmap, case.n, case.hold, entry=entry)
    try:
        case(am, p)
    finally:
        p.close()


# ---- 2. random walks: sparse and dense posts, reads in between, the holds and timeouts, every entry point ---------------
STEPS = [1, 1, 59, 1, 60, 2, 1, -60, 0, 1, 17, 1, 59, 1, 600, 1, 43, 1, -1, 120, 1, 30, 29, 1, 3617, 1, 5, 55, 1]


def _walk(am, zmap, hold, early, mode, seed_text, n=3000):
    rng = np.random.default_rng(zlib.crc32(seed_text.encode()))
    T = M0 + 12 * DAY + 14 * 3600 - 3
    tz = zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))

    def records(k):
        r = am.columns_to_records(population(rng, k, T, True, tz))
        if hold == "remedy":
            r["wf_timeout"] = np.where(rng.random(k) < 0.2, 0, rng.integers(1, 120, k))
        return r

    old = os.environ.get("AMSWEEP_EARLY_RESULTS")
    os.environ["AMSWEEP_EARLY_RESULTS"] = str(early)
    try:
        p = pair(am, zmap, n, hold)
    finally:
        if old is None:
            del os.environ["AMSWEEP_EARLY_RESULTS"]
        else:
            os.environ["AMSWEEP_EARLY_RESULTS"] = old
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
                ph = rng.integers(0, 3, len(sl)).astype(np.uint8)
                rp = np.where(rng.random(len(sl)) < 0.5, 0, rng.integers(1, 3, len(sl))).astype(np.uint8)
                p.post(sl, ph, rp)
                if k % 3 == 1:  # a read between the post and the tick leaves the results pending
                    p.read(rng.choice(n, 10, replace=False))
                    if rng.random() < 0.5:
                        p.post(sl[:20], np.full(20, 1, np.uint8))
            T += step
            p.tick(T, mode, entry=entries[k % len(entries)])
        return p.listed
    finally:
        p.close()


@pytest.mark.parametrize("early", [1, 0], ids=["early_results", "in_sweep"])
@pytest.mark.parametrize("hold", [None, "hold", "remedy"])
@pytest.mark.parametrize("mode", [0, CATCH | FULL], ids=["plain", "catch_up_full"])
def test_random_walks_equal_the_oracle(am, zmap, hold, early, mode):
    listed = _walk(am, zmap, hold, early, mode, f"changes {hold} {early} {mode}")
    assert listed > 1000, listed


def test_closed_loop(am, zmap):
    """every record submitted in closed loop completes in its tick; parse errors emit every tick and change nothing"""
    n = 4000
    rng = np.random.default_rng(5)
    T = M0 + 3
    p = pair(am, zmap, n)
    try:
        p.upsert(np.arange(n), am.columns_to_records(population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY)))))
        for k, step in enumerate([0, 1, 57, 60, 1, 3600]):
            T += step
            if k % 2:
                sl = rng.choice(n, 300, replace=False)
                p.post(sl, rng.integers(0, 3, 300).astype(np.uint8), rng.integers(0, 3, 300).astype(np.uint8))
            p.tick(T, CLOSED | (FULL if k == 2 else 0) | (CATCH if k == 4 else 0), entry=ENTRIES[k % 4])
        assert p.listed > 500, p.listed
    finally:
        p.close()


# ---- 3. catch-up ticks on named zones (amgen config 22) -----------------------------------------------------------------
def test_catch_up_on_named_zones(am, zmap):
    n = 20_000
    T = amgen.T0_MON_0915
    cols = amgen.fill(22, 2, 0, n, T, am.load().am_healthcheck_classify)
    rng = np.random.default_rng(22)
    cols["flags"] |= np.where(rng.random(n) < 0.5, am.F_HAS_REMEDY, 0).astype(np.uint32)
    p = pair(am, zmap, n, "remedy")
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
        assert p.listed > 5000, p.listed
    finally:
        p.close()


# ---- 4. the call contract ----------------------------------------------------------------------------------------------
def test_contract(am, zmap):
    """offset / cap / AM_E_NOSPACE / AM_E_RANGE, NULL columns, refused and AM_E_NOSPACE ticks, run_ticks, the switch"""
    n = 64
    with am.Sweep(capacity=n, shard_base=1000) as s:
        lib = s._lib
        import ctypes as C
        cnt = am.abi.u64(0)
        assert lib.am_sweep_last_changes(s._h, 0, None, None, 0, C.byref(cnt)) == am.AM_E_INVAL  # tracking off
        s.set_track_changes(True)
        assert s.last_changes()[0].tolist() == []  # no tick yet
        recs = np.concatenate([rec(am, 0, repeat_after_sec=60, finished_at=M0 - 10)] * 10 + [rec(am, 0, repeat_after_sec=0)])
        s.upsert(np.arange(11), recs)
        s.post_result(np.arange(10), np.full(10, 1, np.uint8))
        with pytest.raises(am.AmError) as e:  # (slot 10 is reported STOPPED)
            s.tick(M0, cap=0)
        assert e.value.code == am.AM_E_NOSPACE
        idx, cols = s.last_changes(names=["success", "finished_at"])
        assert idx.tolist() == list(range(1000, 1011)) and sorted(cols) == ["finished_at", "success"]
        assert cols["success"].tolist() == [1] * 10 + [0] and (cols["finished_at"] == M0).all()
        # offset / cap
        idx, _ = s.last_changes(offset=7)
        assert idx.tolist() == [1007, 1008, 1009, 1010]
        out = np.zeros(4, np.uint64)
        assert lib.am_sweep_last_changes(s._h, 3, out.ctypes.data, None, 4, C.byref(cnt)) == am.AM_E_NOSPACE
        assert cnt.value == 8 and out.tolist() == [1003, 1004, 1005, 1006]
        assert lib.am_sweep_last_changes(s._h, 11, None, None, 0, C.byref(cnt)) == am.AM_OK and cnt.value == 0
        assert lib.am_sweep_last_changes(s._h, 12, None, None, 0, C.byref(cnt)) == am.AM_E_RANGE
        # a refused tick leaves the list in place
        with pytest.raises(am.AmError):
            s.tick(M0 + 2 * DAY, mode=CATCH)
        assert len(s.last_changes()[0]) == 11
        # a later tick starts a new list, a result left pending by a read included
        s.post_result([4], [2])
        s.read([4])
        s.tick(M0 + 1)
        idx, cols = s.last_changes()
        assert idx.tolist() == [1004] and cols["failed"].tolist() == [1]
        # run_ticks empties the list and tracks nothing
        s.post_result([5], [1])
        s.run_ticks(M0 + 2, 3)
        assert s.last_changes()[0].tolist() == []
        s.tick(M0 + 5)
        assert s.last_changes()[0].tolist() == []
        # off: AM_E_INVAL; on again: a fresh set, which counts results pending before it
        s.post_result([6], [2])
        s.set_track_changes(False)
        s.read([6])
        assert lib.am_sweep_last_changes(s._h, 0, None, None, 0, C.byref(cnt)) == am.AM_E_INVAL
        s.set_track_changes(True)
        assert s.last_changes()[0].tolist() == []
        s.tick(M0 + 6)
        assert s.last_changes()[0].tolist() == [1006]


# ---- 5. random call sequences through the sequence model ------------------------------------------------------------------
class ChangesWalk(Walk):
    """tests/test_call_sequences_gpu.py's walk with tracking on (it compares the changed set after every tick and
    run_ticks); the switch is turned off and on again now and then"""

    def __init__(self, *a, details=False):
        super().__init__(*a, track=True, details=details)
        self.checked = 0

    def tick(self, T, mode, every_column, entry=None):
        if self.step % 11 == 10 and self.rng.integers(0, 2):
            self.set_track()
        self.checked += 1
        return super().tick(T, mode, every_column, entry)


@pytest.mark.parametrize("k", [0, 2, 3, 5], ids=[WALKS[k][3] for k in (0, 2, 3, 5)])
def test_random_call_sequences(am, zmap, k):
    cap, base, T0, name = WALKS[k]
    walk = ChangesWalk(am, zmap, name, zlib.crc32(f"changes {name}".encode()), cap, base, T0)
    walk.run()
    assert walk.checked > 20


# ---- 6. launch counts ----------------------------------------------------------------------------------------------------
def test_launch_counts(am):
    """a handle with tracking off launches what an untracked handle launches, also after on -> off"""
    n = 3000
    recs = np.concatenate([rec(am, 0, repeat_after_sec=60, finished_at=M0 - 100, has_remedy=True)] * n)
    with am.Sweep(capacity=n) as a, am.Sweep(capacity=n) as b, am.Sweep(capacity=n) as c:
        b.set_track_changes(True)
        b.set_track_changes(False)
        counts = {id(s): [] for s in (a, b, c)}
        for k, t in enumerate([M0, M0 + 1, M0 + 30, M0 + 60, M0 + 61]):
            if k == 0:
                for s in (a, b, c):
                    s.upsert(np.arange(n), recs)
            if k == 3:
                c.set_track_changes(True)
            sl = np.arange(0, n, 7 if k % 2 else 2)  # sparse and dense posts
            for s in (a, b, c):
                l0 = s.launch_count
                s.post_result(sl, np.full(len(sl), 2, np.uint8))
                s.read([1])
                s.tick(t)
                counts[id(s)].append(s.launch_count - l0)
        assert counts[id(a)] == counts[id(b)], counts
        # on: the drain's pass over the ops, and after the sweep the exceptions, count, scan and list
        assert [x - y for x, y in zip(counts[id(c)], counts[id(a)])][3:] == [5, 5], counts


# ---- 7. full size, on the GPU only -----------------------------------------------------------------------------------------
def test_full_size_config3(am, zmap):
    """one 10 M-record config 3 tick: 75 % of the records have a result (the dense route), compared in full"""
    if emulated(am):
        pytest.skip("10 M records: GPU only")
    n = 10_000_000
    T0 = amgen.T0_MON_0915
    cols = amgen.fill(3, 3, 0, n, T0, am.load().am_healthcheck_classify)
    with am.Sweep(capacity=n) as s:
        s.set_track_changes(True)
        s.load_range(0, cols)
        before = changes_oracle.snapshot(cols)
        idx, act, _ = zmap.sweep(cols, T0)
        want = changes_oracle.changed(before, cols, idx, act)
        s.tick_view(T0)
        assert len(want) > 7_000_000, len(want)
        check_changes(s, want, cols, "config 3", names=STATUS)
