"""Random call sequences through every entry point of a sweep handle, compared after every call with one sequential
model (tests/handle_model.py): upserts with duplicate slots that flip kinds and zones, removes, sparse and dense
posts (some from four threads), calls past the 32 K-op copy chunk, loads at ragged offsets over slots with staged
calls, the hold turned on and off, every query, and ticks through am_sweep_tick (short buffers and last_list
included), _tick_view, _tick_device (the handle's stream, a torch stream, the default stream), _tick_shard and
run_ticks (blocked and not), plain, full-scan, closed-loop and catch-up, with the clock stepped forwards, twice on one
second and backwards.  Plus the regression test of a load that follows staged calls.

SEQ_CAPACITIES (comma-separated) replaces the handle capacities of the walks (the emulated library runs smaller ones,
tests/test_call_sequences_emulator.py)."""
import os
import threading
import zlib

import numpy as np
import pytest

import oracle_c
from adversarial import MONROVIA, ZoneMap, first_difference, oracle_lookup, population, zones_usable
from handle_model import NONE, HandleModel, Refused
from handle_pair import DevOut, check_changes, check_details, emulated

pytestmark = pytest.mark.gpu

DAY, HOUR = 86400, 3600
FULL, CLOSED, CATCH, BLOCKED = 0x2, 0x1, 0x8, 0x4
BASE_HI = (1 << 32) - 40_000
CHUNK = 32 * 1024  # ops per copy chunk of the staging arrays (kFlushOps)


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def _interval(am, n, ras, fa):
    rc, r = am.classify(repeat_after_sec=ras, finished_at=fa)
    assert rc == 0
    return np.repeat(r, n)


def _cron(am, n, spec):
    rc, r = am.classify(cron=spec)
    assert rc == 0
    return np.repeat(r, n)


# ---- 1. a load is a call in the per-slot order ---------------------------------------------------------------------
@pytest.mark.parametrize("case", ["probe", "probe_hold", "plane_segment"])
def test_load_range_after_staged_calls(am, zmap, case):
    """calls staged before am_sweep_load_range take effect before it: the load wins over every one of them"""
    T = 1790812800 + 7 * HOUR
    if case in ("probe", "probe_hold"):
        A = am.records_to_columns(_interval(am, 8, 60, T - 60))        # due at T
        B = _interval(am, 1, 60, T)                                    # not due at T
        m = HandleModel(zmap, 8)
        with am.Sweep(capacity=8) as s:
            if case == "probe_hold":
                s.set_hold_in_flight(True)
                m.set_hold(True)
                # submitted at T - 60 and held since
                A["finished_at"][:] = T - 120
                s.load_range(0, A)
                m.load(0, A)
                assert len(s.tick(T - 60)[0]) == len(m.tick(T - 60, 0)[0]) == 8
                assert (s.in_flight(0, 8) == T - 60).all()
                A["finished_at"][:] = T - 60
            else:
                s.load_range(0, A)
                m.load(0, A)
            s.upsert([0], B)
            s.remove([1])
            s.post_result([2], [am.PHASE_FAILED])
            m.upsert([0], B)
            m.remove([1])
            m.post([2], [am.PHASE_FAILED])
            if case == "probe_hold":  # not loaded again: the result stays, and it releases the hold
                s.post_result([4], [am.PHASE_SUCCEEDED])
                m.post([4], [am.PHASE_SUCCEEDED])
            three = {k: v[:3].copy() for k, v in A.items()}
            s.load_range(0, three)
            m.load(0, three)
            if case == "probe_hold":  # the load releases 0..2, the posted phase 4; 3 and 5..7 stay held
                f = s.in_flight(0, 8)
                assert f.tolist() == [NONE] * 3 + [T - 60, NONE] + [T - 60] * 3, f
                np.testing.assert_array_equal(f, m.in_flight(0, 8))
            got = s.tick(T)
            want = m.tick(T, 0)
            dev = s.read_range(0, 8)
        idx, act, st = got
        assert idx.tolist() == ([0, 1, 2] if case == "probe_hold" else list(range(8))), idx.tolist()
        assert (act == am.ACT_SUBMIT_HC).all()
        assert st["n_result_fail"] == 0 and st["n_result_ok"] == (case == "probe_hold"), st
        assert first_difference(am, got, want[:3], dev, m.cols()) is None
        for name in am.COLUMN_NAMES:  # three fresh copies of A
            np.testing.assert_array_equal(dev[name][:3], three[name], err_msg=name)
    else:
        # 256 slots = two 128-record plane segments; every minute in UTC, on-minute ticks read the planes
        n = 256
        T = (T // 60) * 60
        every = am.records_to_columns(_cron(am, n, "* * * * *"))
        paris = _cron(am, 11, "CRON_TZ=Europe/Paris 30 3 * * *")  # another kind and zone, not due at T
        quiet = _interval(am, 4, 3600, T)
        m = HandleModel(zmap, n)
        with am.Sweep(capacity=n) as s:
            s.load_range(0, every)
            m.load(0, every)
            s.upsert(np.arange(130, 141), paris)
            m.upsert(np.arange(130, 141), paris)
            s.upsert([150, 151, 200, 129], quiet)
            m.upsert([150, 151, 200, 129], quiet)
            part = {k: v[133:153].copy() for k, v in every.items()}
            s.load_range(133, part)  # the middle of the second segment, over the flipped slots
            m.load(133, part)
            for t in (T, T + 60):
                gi, ga, gs = s.tick(t)
                wi, wa, ws = m.tick(t, 0)[:3]
                assert gs == ws, (t, gs, ws)
                np.testing.assert_array_equal(gi, wi)
                np.testing.assert_array_equal(ga, wa)
            assert {130, 131, 132, 129, 200}.isdisjoint(gi.tolist()) and {133, 140, 150, 151, 152} <= set(gi.tolist())
            got = s.read_range(0, n)
            for name in am.COLUMN_NAMES:
                np.testing.assert_array_equal(got[name], m.cols()[name], err_msg=name)


def test_a_tick_shard_without_an_exchange_leaves_no_statistics(am, zmap):
    """the statistics a tick_shard accumulates are published by the exchange; a host tick that reuses the buffer set
    without one counts only its own"""
    T = 1790812800 + 7
    recs = _interval(am, 64, 3600, T - 10)
    m = HandleModel(zmap, 64)
    with am.Sweep(capacity=64) as s:
        for c in (s, m):
            c.upsert(np.arange(64), recs)
            (c.post_result if c is s else c.post)(np.arange(40), np.ones(40, np.uint8))
        s.tick_shard(T)
        m.tick(T, 0)
        for k in (1, 2, 3):
            assert s.tick(T + k)[2] == m.tick(T + k, 0)[2], k


# ---- 2. random walks -----------------------------------------------------------------------------------------------
# (capacity, shard base, first second, walk name).  Each walk starts before a daylight transition of a zone its records
# are bound to; one runs in Africa/Monrovia's 1971 (UTC-0:44:30: the local minute is not the UTC one).
T_PARIS = 1792890000        # 2026-10-25 01:00 UTC: Europe/Paris leaves summer time
T_NEW_YORK = 1793512800     # 2026-11-01 06:00 UTC: America/New_York leaves daylight time
T_LORD_HOWE = 1791041400    # 2026-10-03 15:30 UTC: Australia/Lord_Howe moves 30 minutes forward
T_NY_1971 = 41410800        # 1971-04-25 07:00 UTC: America/New_York enters daylight time
WALKS = [
    (1, 0, T_PARIS - 400, "one_slot"),
    (1025, BASE_HI, T_NEW_YORK - 700, "base_hi"),
    (8193, 0, T_LORD_HOWE - 500, "lord_howe"),
    (70_001, BASE_HI, T_PARIS - 900, "large_base_hi"),
    (1025, 0, T_NY_1971 - 600, "monrovia_1971"),
    (8193, BASE_HI, T_NEW_YORK - 300, "new_york"),
]
STEPS = [0, 1, -1, 59, 60, 3617, -60]
MODES = [0, FULL, CLOSED, CATCH, CATCH | FULL, CLOSED | FULL, CLOSED | CATCH, CLOSED | CATCH | FULL]
N_STEPS = 36
FORCE_NOSPACE = (12, 29)  # steps whose tick has an empty host buffer (the hold is off at both)


def _capacity(k, cap):
    env = os.environ.get("SEQ_CAPACITIES")
    return int(env.split(",")[k]) if env else cap


class Walk:
    """one handle and its model, driven by one seeded generator; every check names (walk, seed, step, call).  With
    `track` (and `details`) on, every tick and run_ticks also compares the changed set (and the details)."""

    def __init__(self, am, zmap, name, seed, capacity, base, T0, track=False, details=False):
        self.am, self.zmap, self.name, self.seed = am, zmap, name, seed
        self.rng = np.random.default_rng(seed)
        self.n = capacity
        self.T = T0
        self.zones = zones_usable(T0 - DAY, T0 + 2 * DAY)
        self.tz_ids = zmap.ids_of(self.zones)
        self.s = am.Sweep(capacity=capacity, shard_base=base)
        self.m = HandleModel(zmap, capacity, base, seed=seed)
        self.s.set_seed(seed)
        self.details = details
        if track:
            self.set_track()
        self.dev = DevOut(am, capacity)
        self.step = 0
        self.call = "create"
        self.streams = ["handle"] if emulated(am) else ["handle", "torch", "default"]
        self.torch_stream = None
        self.calls = {}
        self.reached = dict(held=0, catch_up_minutes=0, nospace=0, dense_posts=0, zone_transitions=0, big_calls=0)

    @property
    def where(self):
        return (self.name, self.seed, self.step, self.call)

    def note(self, call):
        self.call = call
        self.calls[call] = self.calls.get(call, 0) + 1

    def records(self, k):
        return self.am.columns_to_records(population(self.rng, k, self.T, True, self.tz_ids))

    def slots(self, k):
        return self.rng.integers(0, self.n, k)

    # ---- staged calls ----
    def upsert(self, k=None):
        k = k or int(self.rng.integers(1, min(self.n, 300) + 1))
        sl = self.slots(k)
        if k > 1:  # duplicates within the call: the later entry wins
            sl[-1] = sl[0]
        recs = self.records(k)
        self.note("upsert")
        self.s.upsert(sl, recs)
        self.m.upsert(sl, recs)

    def remove(self):
        sl = self.slots(int(self.rng.integers(1, min(self.n, 60) + 1)))
        self.note("remove")
        self.s.remove(sl)
        self.m.remove(sl)

    def post(self, dense=False, k=None, threads=1):
        hwm = max(self.m.hwm, 1)
        if k is None:
            k = int(self.rng.integers(hwm // 8 + 1, hwm + 2)) if dense else int(self.rng.integers(1, max(hwm // 8, 1) + 1))
        if threads > 1:  # disjoint slots, one call per thread, concurrently
            parts = np.array_split(self.rng.permutation(hwm)[:min(k, hwm)], threads)
        else:
            parts = [self.rng.integers(0, hwm, k)]
        phases = [self.rng.integers(0, 3, len(p)).astype(np.uint8) for p in parts]
        rphases = [self.rng.integers(0, 3, len(p)).astype(np.uint8) for p in parts]
        total = sum(len(p) for p in parts)
        if total * 8 > hwm:
            self.reached["dense_posts"] += 1
        self.note(f"post{'_threads' if threads > 1 else ''}")
        if threads > 1:
            ts = [threading.Thread(target=self.s.post_result, args=(p, ph, rp)) for p, ph, rp in zip(parts, phases, rphases)]
            for t in ts:
                t.start()
            for t in ts:
                t.join()
        else:
            self.s.post_result(parts[0], phases[0], rphases[0])
        for p, ph, rp in zip(parts, phases, rphases):
            self.m.post(p, ph, rp)

    def big_call(self):
        """one call of more ops than a copy chunk holds (duplicate slots on small handles)"""
        k = CHUNK + 7_300
        self.reached["big_calls"] += 1
        if self.rng.integers(0, 2):
            self.post(k=k)
        else:
            sl = self.slots(k)
            recs = np.repeat(self.records(64), k // 64 + 1)[:k]
            self.note("upsert_big")
            self.s.upsert(sl, recs)
            self.m.upsert(sl, recs)

    def load(self, over_staged=False):
        k = int(self.rng.integers(1, min(self.n, 400) + 1))
        first = int(self.rng.integers(0, self.n - k + 1))
        if over_staged and self.n > 1:  # stage calls on slots of the range first
            sl = first + self.rng.integers(0, k, min(k, 8))
            recs = self.records(len(sl))
            self.s.upsert(sl, recs)
            self.m.upsert(sl, recs)
            self.s.remove(sl[:2])
            self.m.remove(sl[:2])
            ph = np.ones(len(sl), np.uint8)
            self.s.post_result(sl, ph)
            self.m.post(sl, ph)
        cols = population(self.rng, k, self.T, True, self.tz_ids)
        self.note("load_range_over_staged" if over_staged else "load_range")
        self.s.load_range(first, cols)
        self.m.load(first, cols)

    def set_hold(self, on):
        self.note("hold_on" if on else "hold_off")
        self.s.set_hold_in_flight(on)
        self.m.set_hold(on)

    def set_track(self):
        """tracking on (again: off first), with details if the walk has them: an empty changed set"""
        for on in ([False, True] if self.m.track else [True]):
            self.s.set_track_changes(on)
            self.m.set_track(on)
        if self.details:
            self.s.set_change_details(True)
            self.m.set_details(True)

    # ---- queries (each drains the staged calls) ----
    def read(self):
        if self.rng.integers(0, 2):
            first = int(self.rng.integers(0, self.n))
            k = int(self.rng.integers(1, self.n - first + 1))
            self.note("read_range")
            got = self.s.read_range(first, k)
            sl = np.arange(first, first + k)
        else:
            sl = self.slots(int(self.rng.integers(1, 50)))
            self.note("read_idx")
            got = self.s.read(sl)
        live = self.m.live(sl)
        for c in self.am.COLUMN_NAMES:
            keep = live | (c == "flags")
            np.testing.assert_array_equal(got[c][keep], self.m.cols()[c][sl][keep], err_msg=f"{self.where} {c}")

    def in_flight(self):
        if self.rng.integers(0, 2):
            first = int(self.rng.integers(0, self.n))
            k = int(self.rng.integers(1, self.n - first + 1))
            self.note("in_flight")
            got, want = self.s.in_flight(first, k), self.m.in_flight(first, k)
        else:
            sl = self.slots(int(self.rng.integers(1, 50)))
            self.note("in_flight_idx")
            got, want = self.s.in_flight(idx=sl), self.m.in_flight(idx=sl)
        np.testing.assert_array_equal(got, want, err_msg=str(self.where))

    def repeat_after(self):
        first = int(self.rng.integers(0, self.n))
        k = int(self.rng.integers(1, min(self.n - first, 48) + 1))
        T = self.T + int(self.rng.integers(-90, 91))
        self.note("repeat_after_sec")
        np.testing.assert_array_equal(self.s.repeat_after_sec(T, first, k), self.m.repeat_after(T, first, k),
                                      err_msg=str((self.where, T, first, k)))

    def next_due(self):
        self.note("next_due")
        nd = self.s.next_due(self.T)
        horizon = 900 if self.m.hwm <= 10_000 else 120
        first = self.m.first_active_tick(self.T, horizon)
        if self.m.live_zone_schedules():  # the next UTC minute (or T + 1) stands in for a zone's schedule
            assert nd is not None and nd > self.T, (self.where, nd)
            assert first is None or nd <= first, (self.where, nd, first)
        elif first is not None:
            assert nd == first, (self.where, nd, first)
        else:
            assert nd is None or nd > self.T + horizon, (self.where, nd)

    # ---- ticks ----
    def _offsets(self, t):
        lib = oracle_c.load()
        import ctypes as C
        out = []
        for z in self.zones:
            o = C.c_int32()
            lib.orc_tz_offset(oracle_lookup(z), t, C.byref(o))
            out.append(o.value)
        return out

    def compare(self, got, want, every_column):
        gi, ga, gs = got
        wi, wa, ws = want[:3]
        assert gs == ws, (self.where, {k: (gs[k], ws[k]) for k in gs if gs[k] != ws[k]})
        np.testing.assert_array_equal(gi, wi, err_msg=str(self.where))
        np.testing.assert_array_equal(ga, wa, err_msg=str(self.where))
        self.check_columns(every_column)

    def check_columns(self, every_column):
        hwm = self.m.hwm
        names = self.am.COLUMN_NAMES if every_column else ["flags", "finished_at", "success", "failed",
                                                             "remedy_success", "remedy_failed", "remedy_total",
                                                             "remedy_finished_at"]
        got = self.s.read_range(0, hwm, names)
        live = self.m.live(np.arange(hwm))
        for c in names:
            want = self.m.cols()[c]
            bad = np.flatnonzero((got[c] != want[:hwm]) & (live | (c == "flags")))
            assert len(bad) == 0, (self.where, c, int(bad[0]), int(got[c][bad[0]]), int(want[bad[0]]))
        if every_column:
            np.testing.assert_array_equal(self.s.in_flight(0, self.n), self.m.in_flight(0, self.n), err_msg=str(self.where))

    def tick(self, T, mode, every_column, entry=None):
        am, s, m = self.am, self.s, self.m
        self.reached["held"] += int(m.held().sum())
        P = m.window_of(T, mode)
        if P is not None and T - P <= DAY and any(t % 60 == 0 for t in range(P + 1, T + 1)):
            self.reached["catch_up_minutes"] += 1
        if m.P is not None and self._offsets(m.P) != self._offsets(T):
            self.reached["zone_transitions"] += 1
        entry = entry or str(self.rng.choice(["tick", "tick", "tick_short", "tick_view", "tick_device", "tick_shard"]))
        self.note(entry)
        try:
            want = m.tick(T, mode)
        except Refused as r:
            before = s.launch_count
            with pytest.raises(am.AmError) as e:
                self._call(entry, T, mode, None)
            assert e.value.code == r.code, (self.where, e.value.code, r.code)
            assert s.launch_count == before, self.where
            self.check_lists(False)
            return False
        self.device_cap = None
        got = self._call(entry, T, mode, want)
        self.reached["held"] += int(m.held().sum())  # submitted by this tick and held from now on
        if got is None:  # tick_shard: the list stays on the device
            self.check_columns(True)
        else:
            if self.device_cap is not None:  # a short device buffer holds the list's first cap entries
                want = (want[0][:self.device_cap], want[1][:self.device_cap], want[2])
            self.compare(got, want, every_column)
        self.check_lists(True)
        return True

    def check_lists(self, ticked):
        """the changed set with tracking on (its columns after a tick), the details with details on"""
        m, s = self.m, self.s
        if m.track and ticked:
            check_changes(s, m.changes(), m.cols(), self.where)
        elif m.track:
            np.testing.assert_array_equal(s.last_changes(names=[])[0], m.changes(), err_msg=str(self.where))
        if m.details_on:
            det = m.details()
            check_details(s, m.changes() if len(det) else np.zeros(0, np.uint64), det, self.where)

    def _call(self, entry, T, mode, want):
        am, s = self.am, self.s
        if entry == "tick":
            return s.tick(T, mode=mode)
        if entry == "tick_short":
            cap = 0 if self.step in FORCE_NOSPACE else int(self.rng.integers(0, 6))
            try:
                got = s.tick(T, mode=mode, cap=cap)
                return got
            except am.AmError as e:
                if e.code != am.AM_E_NOSPACE:
                    raise
                self.reached["nospace"] += 1
                gi, ga, gs = e.partial
                assert e.needed == gs["n_emitted"] > cap, self.where
                parts_i, parts_a, off = [gi[:cap]], [ga[:cap]], cap
                while off < e.needed:  # the rest in pieces
                    piece = int(self.rng.integers(1, max(e.needed // 3, 1) + 1))
                    i, a, left = s.last_list(off, piece)
                    assert left == e.needed - off, self.where
                    parts_i.append(i)
                    parts_a.append(a)
                    off += len(i)
                return np.concatenate(parts_i), np.concatenate(parts_a), gs
        if entry == "tick_view":
            i, a, st = s.tick_view(T, mode=mode)
            return i.astype(np.uint64) + np.uint64(s.shard_base), a.astype(np.uint32), st
        if entry == "tick_device":
            which = str(self.rng.choice(self.streams))
            if which == "torch":
                import torch
                self.torch_stream = self.torch_stream or torch.cuda.Stream()
                stream = self.torch_stream.cuda_stream
            else:
                stream = s.stream if which == "handle" else 0
            self.note(f"tick_device_{which}")
            cap = self.n if self.rng.integers(0, 3) else int(self.rng.integers(0, 8))
            self.device_cap = cap
            return self.dev.tick(am, s, T, mode, cap, stream)
        s.tick_shard(T, mode=mode)
        return None

    def run_ticks(self, T, every_column):
        am, s, m = self.am, self.s, self.m
        k = int(self.rng.integers(1, 140))
        mode = int(self.rng.choice([0, FULL, CLOSED, BLOCKED, BLOCKED | CLOSED, BLOCKED | FULL, CATCH]))
        block = str(self.rng.choice(["7", "96"]))
        seed = int(self.rng.integers(0, 1 << 40))
        self.note(f"run_ticks{'_blocked' if mode & BLOCKED else ''}")
        old = os.environ.get("AMSWEEP_BLOCK_TICKS")
        os.environ["AMSWEEP_BLOCK_TICKS"] = block
        try:
            try:
                want = m.run_ticks(T, k, mode, seed)
            except Refused as r:
                before = s.launch_count
                with pytest.raises(am.AmError) as e:
                    s.run_ticks(T, k, mode=mode, seed=seed)
                assert e.value.code == r.code and s.launch_count == before, self.where
                self.check_lists(False)
                return 0
            got = s.run_ticks(T, k, mode=mode, seed=seed)
        finally:
            if old is None:
                del os.environ["AMSWEEP_BLOCK_TICKS"]
            else:
                os.environ["AMSWEEP_BLOCK_TICKS"] = old
        for j in range(k):
            row = {f: int(got[j][f]) for f in am.abi.STAT_FIELDS}
            assert row == want[j], (self.where, j, {f: (row[f], want[j][f]) for f in row if row[f] != want[j][f]})
        self.check_columns(every_column)
        self.check_lists(False)
        return k

    # ---- the walk ----
    def run(self):
        rng = self.rng
        self.note("load_range")
        cols = population(rng, self.n, self.T, True, self.tz_ids)
        self.s.load_range(0, cols)
        self.m.load(0, cols)
        stagers = [self.upsert, self.remove, self.post, lambda: self.post(dense=True), lambda: self.post(threads=4),
                   self.load, lambda: self.load(over_staged=True), self.read, self.in_flight, self.repeat_after,
                   self.next_due]
        for self.step in range(N_STEPS):
            entry = None
            if self.step in (2, 18, 31):
                self.set_hold(True)
            elif self.step == 3:
                self.big_call()
            elif self.step in (11, 27):
                self.set_hold(False)
            for _ in range(int(rng.integers(0, 5))):
                stagers[int(rng.integers(0, len(stagers)))]()
            if self.step in (2, 18, 31) + FORCE_NOSPACE:  # a check that is due at once, into a random slot
                sl = self.slots(1)
                recs = _interval(self.am, 1, 60, self.T - 100)
                self.note("upsert")
                self.s.upsert(sl, recs)
                self.m.upsert(sl, recs)
                if self.step in FORCE_NOSPACE:
                    entry = "tick_short"
            if self.step % 9 == 5:  # a dense post and a load over staged slots in every walk
                self.post(dense=True)
                self.load(over_staged=True)
            every_column = self.step % 5 == 0
            if self.step % 7 == 6:
                self.T += self.run_ticks(self.T + 1, every_column)
                continue
            step = int(rng.choice(STEPS, p=[0.1, 0.3, 0.05, 0.2, 0.2, 0.08, 0.07]))
            mode = int(rng.choice(MODES))
            if self.m.hold and (rng.integers(0, 3) or self.step in (2, 18, 31)):  # (refused while the hold is on)
                mode &= ~CLOSED
            if self.step == 8:  # a day and a second: a catch-up tick is refused
                step, mode = DAY + 1, CATCH
            elif self.step == 9:
                step = 3617
            elif self.step in (4, 14, 24):  # the ticker's cadence across minute starts, catching up
                step, mode = 60 - (self.T % 60) + int(rng.integers(0, 5)), CATCH | (mode & FULL)
            if self.tick(self.T + step, mode, every_column, entry):
                self.T += step
        self.s.close()
        return self.calls, self.reached


@pytest.mark.parametrize("rep", [0, 1])
@pytest.mark.parametrize("k", range(len(WALKS)), ids=[w[3] for w in WALKS])
def test_random_call_sequences_equal_the_model(am, zmap, k, rep):
    cap, base, T0, name = WALKS[k]
    cap = _capacity(k, cap)
    seed = zlib.crc32(f"{name} {rep}".encode())
    T0 += 37 * rep
    walk = Walk(am, zmap, name, seed, cap, base, T0)
    if name == "monrovia_1971":
        assert MONROVIA in walk.zones
    calls, reached = walk.run()
    print(f"\n{name}: capacity {cap}, base {base}, seed {seed}: {sum(calls.values())} calls {sorted(calls.items())} "
          f"reached {reached}")
    assert reached["held"] > 0 and reached["catch_up_minutes"] > 0 and reached["nospace"] > 0, reached
    assert reached["dense_posts"] > 0 and reached["zone_transitions"] > 0 and reached["big_calls"] > 0, reached
