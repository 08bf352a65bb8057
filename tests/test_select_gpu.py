"""Sparse state queries (am_sweep_select): for every state, the list, values, count and least value must be the dense
query of the same state filtered on the host — am_sweep_in_flight, am_sweep_remedy_in_flight, am_sweep_deferred — and
the sequential model's (tests/admission_model.py).  Checked after every step of random call sequences that toggle the
holds and the submit budget; at group, capacity and shard-base boundaries with every cap and cursor paging; with calls
staged before the query; for the refusals, the states that are off and the launch counts; across a checkpoint; behind
a tick queued on a caller stream; and, on an H100, at 10 M records after a simulated hour."""
import zlib

import numpy as np
import pytest

import admission_oracle as ao
import hold_oracle
from adversarial import ZoneMap, population, zones_usable
from admission_model import AdmissionModel
from handle_pair import Pair, emulated
from timeout_cases import rec

pytestmark = pytest.mark.gpu

DAY, HOUR = 86400, 3600
T_OCT = 1790812800  # 2026-10-01 00:00:00 UTC
NONE = hold_oracle.NOT_IN_FLIGHT
I64_MAX = (1 << 63) - 1
GROUP = 8192
IN_FLIGHT, REMEDY, WAITING = 1, 2, 3
DENSE = {IN_FLIGHT: "in_flight", REMEDY: "remedy_in_flight", WAITING: "deferred"}


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def expect(dense, first, before, base=0):
    """select's answer over the slots [first, first + len(dense)) as a filter of their dense values"""
    hit = np.flatnonzero((dense != NONE) & (dense <= before))
    v = dense[hit]
    return (hit + first + base).astype(np.uint64), v, len(hit), int(v.min()) if len(v) else I64_MAX


def check(s, state, dense, first, n, before, where, cap=None):
    """s.select over [first, first + n) against `dense` (the dense values of every slot from 0 on)"""
    got = s.select(state, first, n, before, cap)
    wi, wv, wn, wo = expect(dense[first:first + n], first, before, s.shard_base)
    k = wn if cap is None else min(cap, wn)
    what = f"{where}: state {state} [{first}, +{n}) before {before} cap {cap}"
    np.testing.assert_array_equal(got[0], wi[:k], err_msg=what)
    np.testing.assert_array_equal(got[1], wv[:k], err_msg=what)
    assert got[2:] == (wn, wo), (what, got[2:], (wn, wo))
    return wn


def befores(vals, T):
    """a spread of bounds: everything, nothing, the least, median and greatest value and some below T"""
    out = [I64_MAX, NONE, T - 30]
    v = vals[vals != NONE]
    if len(v):
        out += [int(v.min()), int(np.median(v)), int(v.max()) - 1, int(v.max())]
    return out


def model_values(m, n):
    return {IN_FLIGHT: m.in_flight(0, n), REMEDY: m.remedy_in_flight(0, n), WAITING: m.deferred(0, n)}


class SelPair(Pair):
    """tests/handle_pair.py's Pair with AdmissionModel as the model; select is compared with the model right after
    every tick of the handle (before any other call, so behind a tick on a caller stream) and by check_all"""

    def __init__(self, am, zmap, cols, entry="tick"):
        self.am, self.entry, self.cap, self.every_slot = am, entry, 1, True
        self.n = len(cols["flags"])
        self.s = am.Sweep(capacity=self.n)
        self.m = AdmissionModel(zmap, self.n)
        self.load(0, cols)
        self.dev = None
        self.timed_total = self.rtimed_total = self.started = self.listed = self.detailed = 0
        self.T = 0
        self.matches = {IN_FLIGHT: 0, REMEDY: 0, WAITING: 0}

    def set_budget(self, v):
        self._switch(self.s.set_submit_budget, self.m.set_budget, v)

    def _call(self, entry, T, mode, want):
        got = super()._call(entry, T, mode, want)
        for state, vals in model_values(self.m, self.n).items():
            check(self.s, state, vals, 0, self.n, I64_MAX, f"after the tick at {T} ({entry})")
        return got

    def check_all(self, rng, where):
        """every state against its dense query and the model, at a spread of bounds, over the whole range and over
        one that starts and ends at random slots"""
        want = model_values(self.m, self.n)
        for state, fn in DENSE.items():
            check(self.s, state, want[state], 0, self.n, I64_MAX, where)  # (the first call after staged ones drains)
            dense = getattr(self.s, fn)(0, self.n)
            np.testing.assert_array_equal(dense, want[state], err_msg=f"{where}: {fn}")
            a, b = sorted(rng.integers(0, self.n + 1, 2).tolist())
            for before in befores(dense, self.T):
                self.matches[state] += check(self.s, state, dense, 0, self.n, before, where)
                check(self.s, state, dense, a, b - a, before, where)


def _records(am, rng, n, T, zmap):
    recs = am.columns_to_records(population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY))))
    recs["wf_timeout"] = rng.integers(0, 200, n)
    return recs


STEPS = [1, 1, 59, 1, 1, 60, 1, 2, 1, 57, 1, 0, 1, -30, 1, 600, 1, 1, 60, 1, 1, 59, 1, 1]


@pytest.mark.parametrize("entry", ["tick", "tick_device", "tick_shard"])
def test_random_sequences_equal_the_dense_queries_and_the_model(am, zmap, entry):
    n = 2500
    rng = np.random.default_rng(zlib.crc32(f"select {entry}".encode()))
    T = T_OCT + 9 * DAY + 11 * HOUR - 2
    p = SelPair(am, zmap, population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))), entry=entry)
    toggled = 0
    try:
        p.set_hold(True)
        p.set_remedy(True)
        p.upsert(np.arange(n), _records(am, rng, n, T, zmap))
        p.set_budget(40)
        for k, step in enumerate(STEPS):
            p.T = T
            r = rng.random()
            if k % 8 == 5:  # the hold off and on again: everything ends, the budget is unlimited
                p.set_hold(False)
                p.check_all(rng, f"step {k}: hold off")
                p.set_hold(True)
                p.set_remedy(True)
                toggled += 1
            elif k % 8 == 6:
                p.set_remedy(False)
                p.check_all(rng, f"step {k}: remedy hold off")
                p.set_remedy(True)
            if k % 3 == 0:
                p.set_budget([0, 5, 40, 300, None][int(rng.integers(0, 5))])
            waiting = np.flatnonzero(p.m.wait != ao.NOT_WAITING)
            busy = np.flatnonzero(p.m.since != NONE)
            if r < 0.3:
                sl = rng.choice(n, 30, replace=False)
                p.upsert(sl, _records(am, rng, len(sl), T, zmap))
            elif r < 0.45:
                p.remove(np.concatenate([rng.choice(n, 10, replace=False), waiting[:5]]))
            elif r < 0.55:
                p.load(int(rng.integers(0, n - 100)),
                       population(rng, 100, T, True, zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))))
            sl = np.concatenate([rng.choice(busy, min(len(busy), 60), replace=False), waiting[5:10]])
            if len(sl):
                p.post(sl, rng.integers(1, 3, len(sl)).astype(np.uint8), rng.integers(0, 3, len(sl)).astype(np.uint8))
            p.check_all(rng, f"step {k}: calls staged at {T}")
            T += step
            p.T = T
            p.tick(T)
            p.check_all(rng, f"step {k}: tick at {T}")
        assert toggled >= 2 and all(v > 100 for v in p.matches.values()), p.matches
    finally:
        p.close()


def _interval_handle(am, capacity, T0, shard_base=0):
    """every slot an interval check of 1 s, due at T0, the hold on; after ticks at T0, T0 + 1 and T0 + 2 with every
    third slot's run posted Succeeded before T0 + 1, every slot is in flight: since T0 + 2 for those, T0 for the rest"""
    s = am.Sweep(capacity=capacity, shard_base=shard_base)
    s.set_hold_in_flight(True)
    s.load_range(0, am.records_to_columns(np.concatenate([rec(am, 0, repeat_after_sec=1, finished_at=T0 - 100)]
                                                         * capacity)))
    s.tick(T0)
    third = np.arange(0, capacity, 3)
    s.post_result(third, np.ones(len(third), np.uint8))
    s.tick(T0 + 1)
    s.tick(T0 + 2)
    want = np.full(capacity, T0, np.int64)
    want[third] = T0 + 2
    np.testing.assert_array_equal(s.in_flight(0, capacity), want)
    return s


@pytest.mark.parametrize("shard_base", [0, (1 << 32) + 5], ids=["base_0", "base_past_2^32"])
def test_boundaries_caps_and_paging(am, shard_base):
    cap_slots = 3 * GROUP + 77  # not a multiple of a group
    T0 = T_OCT + 2 * DAY + 600
    rng = np.random.default_rng(7)
    edges = [0, 1, GROUP - 1, GROUP, 2 * GROUP - 1, 2 * GROUP, 3 * GROUP - 1, 3 * GROUP, cap_slots - 1]
    keep = np.unique(np.concatenate([edges, rng.choice(cap_slots, 300, replace=False)]))
    s = _interval_handle(am, cap_slots, T0, shard_base)
    try:
        done = np.setdiff1d(np.arange(cap_slots), keep)
        s.post_result(done, np.ones(len(done), np.uint8))  # staged: the select's drain releases them
        idx, val, nm, old = s.select(IN_FLIGHT)
        np.testing.assert_array_equal(idx, keep.astype(np.uint64) + np.uint64(shard_base))
        assert nm == len(keep) and old == T0
        dense = s.in_flight(0, cap_slots)
        ranges = [(0, cap_slots), (0, 1), (GROUP - 1, 2), (GROUP - 1, 1), (GROUP, 1), (100, GROUP), (8000, 8400),
                  (GROUP - 1, cap_slots - GROUP + 1), (cap_slots - 1, 1), (cap_slots - 78, 78), (5, cap_slots - 10),
                  (2 * GROUP - 1, GROUP + 2), (3 * GROUP, 77)]
        for first, n in ranges:
            for before in (I64_MAX, T0, T0 + 1, T0 - 1, NONE):
                check(s, IN_FLIGHT, dense, first, n, before, "ranges")
        for first, n in ((0, cap_slots), (GROUP - 1, GROUP + 3)):
            m = expect(dense[first:first + n], first, I64_MAX)[2]
            for cap in sorted({0, 1, max(m - 1, 0), m, m + 1, m + 1000}):
                check(s, IN_FLIGHT, dense, first, n, I64_MAX, "caps", cap=cap)
        want = expect(dense, 0, T0 + 2, shard_base)
        for page in (1, 7, 64, 1000):
            got_i, got_v, first = [], [], 0
            while True:
                i, v, nm, _ = s.select(IN_FLIGHT, first, cap_slots - first, T0 + 2, cap=page)
                got_i.append(i)
                got_v.append(v)
                if nm <= page:
                    break
                first = int(i[-1]) - shard_base + 1
            np.testing.assert_array_equal(np.concatenate(got_i), want[0], err_msg=f"page {page}")
            np.testing.assert_array_equal(np.concatenate(got_v), want[1], err_msg=f"page {page}")
        # states that are off: the remedy hold, the admission state
        for state in (REMEDY, WAITING):
            i, v, nm, old = s.select(state)
            assert len(i) == len(v) == 0 and (nm, old) == (0, I64_MAX)
    finally:
        s.close()


def test_staged_calls_are_applied_first(am, zmap):
    """a posted phase releases the run, a remove ends it and an upsert keeps it before the query sees the slot"""
    n = 64
    T0 = T_OCT + 5 * DAY
    s = _interval_handle(am, n, T0)
    try:
        s.post_result([3, 4], [1, 2])
        s.remove([5])
        s.upsert([6], rec(am, 0, repeat_after_sec=7, finished_at=T0 - 100))
        idx, val, nm, old = s.select(IN_FLIGHT)
        want = np.setdiff1d(np.arange(n), [3, 4, 5])
        np.testing.assert_array_equal(idx, want.astype(np.uint64))
        assert nm == n - 3 and old == T0
        s.post_result([7], [1])
        assert s.select(IN_FLIGHT, 7, 1)[2] == 0  # the counting form drains as well
        s.post_result([8], [1])
        assert s.select(IN_FLIGHT, 0, n, cap=0)[2] == n - 5
    finally:
        s.close()


def _raw(am, s, state=IN_FLIGHT, first=0, n=None, before=I64_MAX, cap=0, arrays=True, counts=True):
    import ctypes as C
    n = s.capacity if n is None else n
    nm, old = am.abi.u64(7), am.abi.i64(7)
    idx, val = np.empty(max(cap, 1), np.uint64), np.empty(max(cap, 1), np.int64)
    rc = s._lib.am_sweep_select(s._h, state, first, n, before, idx.ctypes.data if arrays else None,
                                val.ctypes.data if arrays else None, cap, C.byref(nm) if counts else None,
                                C.byref(old) if counts else None)
    return rc, int(nm.value), int(old.value), idx[:cap], val[:cap]


def test_refusals_and_states_that_are_off(am):
    n = 100
    T0 = T_OCT + 6 * DAY
    s = _interval_handle(am, n, T0)
    try:
        s.post_result([1], [1])  # staged: a refusal must not drain it
        l0 = s.launch_count
        for kw in (dict(state=0), dict(state=4), dict(counts=False), dict(cap=3, arrays=False),
                   dict(first=n, n=1), dict(first=1, n=n), dict(first=(1 << 64) - 1, n=2)):
            assert _raw(am, s, **kw)[0] == am.AM_E_INVAL, kw
        assert s.launch_count == l0
        assert s.in_flight(1, 1)[0] == NONE  # (the post was still staged)
        # nothing to look at: no drain, no launch, nothing found
        s.post_result([2], [1])
        l0 = s.launch_count
        assert _raw(am, s, first=n, n=0, cap=4)[:3] == (am.AM_OK, 0, I64_MAX)
        assert s.launch_count == l0
        # states that are off: the drain only
        s.in_flight(0, 1)
        for state in (REMEDY, WAITING):
            l0 = s.launch_count
            assert _raw(am, s, state=state, cap=5)[:3] == (am.AM_OK, 0, I64_MAX)
            assert s.launch_count == l0
        s.set_hold_in_flight(False)
        for state in (IN_FLIGHT, REMEDY, WAITING):
            l0 = s.launch_count
            assert _raw(am, s, state=state, cap=5)[:3] == (am.AM_OK, 0, I64_MAX)
            assert s.launch_count == l0
        # AM_E_NOSPACE: the first cap entries, the whole range's count and least value
        s.set_hold_in_flight(True)
        s.tick(T0 + 10)
        rc, nm, old, idx, val = _raw(am, s, cap=3)
        # (slots 1 and 2 got their posted results at this tick: not due again before T0 + 11)
        assert (rc, nm, old) == (am.AM_E_NOSPACE, n - 2, T0 + 10) and idx.tolist() == [0, 3, 4]
        assert val.tolist() == [T0 + 10] * 3
    finally:
        s.close()


def test_launch_counts(am):
    n = 3 * GROUP + 5
    T0 = T_OCT + 7 * DAY
    a, b = _interval_handle(am, n, T0), _interval_handle(am, n, T0)
    try:
        a.in_flight(0, 1)  # nothing staged from here on
        for cap, before, want in ((10, I64_MAX, 4), (0, I64_MAX, 1), (10, T0 - 1, 4), (0, T0 - 1, 1), (n, I64_MAX, 4)):
            l0 = a.launch_count
            a.select(IN_FLIGHT, 0, n, before, cap)
            assert a.launch_count - l0 == want, (cap, before)
        # a tick launches what it launched before the handle ever selected
        for k in range(3):
            T = T0 + 3 + 60 * k
            for s in (a, b):
                s.post_result(np.arange(0, n, 5), np.ones(len(range(0, n, 5)), np.uint8))
            d = []
            for s in (a, b):
                l0 = s.launch_count
                s.tick(T)
                d.append(s.launch_count - l0)
            assert d[0] == d[1], d
    finally:
        a.close()
        b.close()


def _handle_like(am, info, capacity, shard_base=0):
    t = am.Sweep(capacity=capacity, shard_base=shard_base)
    sw = info["switches"]
    for bit, call in ((am.CKPT_HOLD, t.set_hold_in_flight), (am.CKPT_REMEDY, t.set_hold_remedy)):
        if sw & bit:
            call(True)
    if sw & am.CKPT_ADMISSION:
        t.set_submit_budget(0)
        t.set_submit_budget(None)
    return t


def test_checkpoint_restores_answer_as_the_source(am, zmap):
    """a checkpoint restored into a fresh handle, and cut into two resharded ones, answers every state as the source"""
    n, cut = 3000, 1337
    rng = np.random.default_rng(41)
    T = T_OCT + 4 * DAY + 9 * HOUR + 30
    p = SelPair(am, zmap, population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))))
    handles = []
    try:
        p.set_hold(True)
        p.set_remedy(True)
        p.upsert(np.arange(n), _records(am, rng, n, T, zmap))
        p.set_budget(40)
        for k, step in enumerate([0, 1, 60, 1, 1, 59]):
            T += step
            if k == 3:
                busy = np.flatnonzero(p.m.since != NONE)[:50]
                p.post(busy, rng.integers(1, 3, len(busy)).astype(np.uint8), rng.integers(0, 3, len(busy)).astype(np.uint8))
            p.tick(T)
        src = model_values(p.m, n)
        assert all((v != NONE).sum() > 20 for v in src.values()), {k: int((v != NONE).sum()) for k, v in src.items()}
        blob = p.s.checkpoint()
        t = _handle_like(am, am.checkpoint_info(blob), n)
        t.restore(blob)
        handles.append(t)
        shards = []
        for lo, hi in ((0, cut), (cut, n)):
            part = p.s.checkpoint(lo, hi - lo)
            u = _handle_like(am, am.checkpoint_info(part), hi - lo, shard_base=lo)
            u.restore(part)
            handles.append(u)
            shards.append(u)
        for state, vals in src.items():
            for before in befores(vals, T):
                want = p.s.select(state, 0, n, before)
                got = t.select(state, 0, n, before)
                np.testing.assert_array_equal(got[0], want[0])
                np.testing.assert_array_equal(got[1], want[1])
                assert got[2:] == want[2:]
                check(t, state, vals, 0, n, before, "restored")
                parts = [u.select(state, 0, u.capacity, before) for u in shards]
                np.testing.assert_array_equal(np.concatenate([q[0] for q in parts]), want[0])
                np.testing.assert_array_equal(np.concatenate([q[1] for q in parts]), want[1])
                assert sum(q[2] for q in parts) == want[2] and min(q[3] for q in parts) == want[3]
    finally:
        for h in handles:
            h.close()
        p.close()


def test_caller_stream_tick_is_seen(am):
    """a tick of am_sweep_tick_device queued behind a long kernel on a caller stream: select waits for it, as the
    dense query does"""
    if emulated(am):
        pytest.skip("a caller stream needs the GPU")
    import torch
    n = 2 * GROUP + 3
    T0 = T_OCT + 8 * DAY
    s = _interval_handle(am, n, T0)
    try:
        done = np.arange(0, n, 2)
        s.post_result(done, np.ones(len(done), np.uint8))
        s.tick(T0 + 3)  # applies them: due again at T0 + 4
        assert s.select(IN_FLIGHT, cap=0)[2] == n - len(done)
        d_idx = torch.empty(n, dtype=torch.int32, device="cuda")
        d_act = torch.empty(n, dtype=torch.uint8, device="cuda")
        d_cnt = torch.zeros(4, dtype=torch.int32, device="cuda")
        d_st = torch.zeros(16, dtype=torch.int64, device="cuda")
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            torch.cuda._sleep(200_000_000)  # a long kernel ahead of the tick
            s.tick_device(T0 + 4, 0, d_idx.data_ptr(), d_act.data_ptr(), n, d_cnt.data_ptr(), d_st.data_ptr(),
                          side.cuda_stream)
        idx, val, nm, old = s.select(IN_FLIGHT)
        torch.cuda.synchronize()
        assert nm == n and old == T0 and int((val == T0 + 4).sum()) == len(done)
        np.testing.assert_array_equal(val, s.in_flight(0, n))
    finally:
        s.close()


def test_full_size_simulated_hour(am):
    """10 M config-5 records after a simulated hour with millions of runs in flight: select equals the dense reads"""
    if emulated(am):
        pytest.skip("10 M records: GPU only")
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import run_sim
    n = 10_000_000
    cols, sl, recs = run_sim.population(am, n, run_sim.SEED)
    T = run_sim.amgen.T0_DAY_START
    with am.Sweep(capacity=n) as s:
        s.load_range(0, cols)
        s.set_hold_in_flight(True)
        s.set_hold_remedy(True)
        s.upsert(sl, recs)
        s.simulate(T, 3600, am.SWEEP_BLOCKED, run_sim.SEED, run_sim.PARAMS)
        T += 3600
        for state in (IN_FLIGHT, REMEDY):
            dense = s.in_flight(0, n) if state == IN_FLIGHT else s.remedy_in_flight(0, n)
            if state == IN_FLIGHT:
                assert (dense != NONE).sum() > 1_000_000
            for before in (I64_MAX, T - 300, int(np.median(dense[dense != NONE])) if (dense != NONE).any() else NONE):
                check(s, state, dense, 0, n, before, "10 M")
            check(s, state, dense, 1234567, 5_000_000, T - 60, "10 M, mid-range")
