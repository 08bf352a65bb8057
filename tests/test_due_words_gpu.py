"""The due words of the open-loop tick (due_word, csrc/sweep_kernels.cuh): a handle that decides interval checks from
them against a twin that has handed out finished_at through am_sweep_column_ptr and so reads ras and finishedAt as
before.  Both see the same seeded calls through every entry point (upserts, spec updates, removes, posts, loads,
restores, delta restores, ticks plain, full-scan and closed-loop, run_ticks blocked and not, the hold on and off), and
after every call their lists, actions, statistics and sixteen columns must be identical; the walks without spec
updates and restores also follow the sequential model (tests/handle_model.py).  Then the cases at the words' edges:
ticks at the ends of the epoch window and just outside it, clamped words, posted phases with ras <= 0 and > 0, unarmed
timers, STOPPED together with a result, results through the drain and through the sweep, a spec edit of ras, a restore
followed by a tick, and a caller's write through the finished_at pointer.

A handle's first open-loop plain tick at T builds the words with the epoch E = T - 2^31; the window is
[E, E + 2^32 - 1).  SEQ_CAPACITIES (comma-separated) replaces the walks' capacities (tests/test_due_words_emulator.py)."""
import ctypes as C
import os

import numpy as np
import pytest

from adversarial import ZoneMap, population, zones_usable
from handle_model import HandleModel
from handle_pair import DevOut, emulated

pytestmark = pytest.mark.gpu

FULL, CLOSED, BLOCKED = 0x2, 0x1, 0x4
T0 = 1789982100  # 2026-09-21 09:15:00 UTC
LEAD = 1 << 31   # T - E of the tick that builds the words
SPAN = (1 << 32) - 1


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def _capacity(k, cap):
    env = os.environ.get("SEQ_CAPACITIES")
    return int(env.split(",")[k]) if env else cap


def _write_column(am, s, name, idx, values):
    """a caller's write of `values` into slots `idx` of column `name` through am_sweep_column_ptr"""
    ptr = s.column_ptr(name)
    dt = np.dtype(dict(am.abi.COLUMNS)[name])
    values = np.ascontiguousarray(values, dtype=dt)
    if emulated(am):
        for i, v in zip(np.asarray(idx).tolist(), values):
            C.memmove(ptr + i * dt.itemsize, v.tobytes(), dt.itemsize)
        return
    import torch

    class _A:
        pass
    a = _A()
    a.__cuda_array_interface__ = {"shape": (s.capacity,), "typestr": dt.str, "data": (ptr, False), "version": 3}
    t = torch.as_tensor(a, device="cuda")
    t[torch.as_tensor(np.asarray(idx, dtype=np.int64), device="cuda")] = torch.as_tensor(values, device="cuda")
    torch.cuda.synchronize()


class Twins:
    """handle `a` (due words), handle `b` (finished_at handed out: never the words) and, optionally, the model"""

    def __init__(self, am, zmap, n, model=True, seed=0):
        self.am, self.n = am, n
        self.a = am.Sweep(capacity=n)
        self.b = am.Sweep(capacity=n)
        self.b.column_ptr("finished_at")
        self.m = HandleModel(zmap, n, seed=seed) if model else None
        for s in (self.a, self.b):
            s.set_seed(seed)
        self.dev = [DevOut(am, n), DevOut(am, n)]
        self.where = None

    def close(self):
        self.a.close()
        self.b.close()

    def both(self, call, *args):
        getattr(self.a, call)(*args)
        getattr(self.b, call)(*args)

    def model(self, call, *args):
        if self.m is not None:
            getattr(self.m, call)(*args)

    def columns(self, what):
        h = self.n
        ca, cb = self.a.read_range(0, h), self.b.read_range(0, h)
        # (the model: flags everywhere, the other columns of live slots; a slot removed in the drain of its upsert keeps
        # stale columns that differ)
        live = self.m.live(np.arange(h)) if self.m is not None else None
        for name in self.am.COLUMN_NAMES:
            np.testing.assert_array_equal(ca[name], cb[name], err_msg=f"{what}: {name}")
            if self.m is not None:
                keep = live | (name == "flags")
                np.testing.assert_array_equal(ca[name][keep], self.m.cols()[name][:h][keep], err_msg=f"{what}: model {name}")

    def tick(self, T, mode=0, entry="tick"):
        what = (self.where, entry, T, mode)
        if entry == "tick_device":
            got = [d.tick(self.am, s, T, mode) for d, s in zip(self.dev, (self.a, self.b))]
        else:
            got = [getattr(s, entry)(T, mode=mode) for s in (self.a, self.b)]
            if entry == "tick_view":
                got = [(i.astype(np.uint64).copy(), x.astype(np.uint32).copy(), st) for i, x, st in got]
        (ia, xa, sa), (ib, xb, sb) = got
        assert sa == sb, (what, {k: (sa[k], sb[k]) for k in sa if sa[k] != sb[k]})
        np.testing.assert_array_equal(ia, ib, err_msg=f"{what}: idx")
        np.testing.assert_array_equal(xa, xb, err_msg=f"{what}: act")
        if self.m is not None:
            want = self.m.tick(T, mode)
            assert sa == want.stats, (what, {k: (sa[k], want.stats[k]) for k in sa if sa[k] != want.stats[k]})
            np.testing.assert_array_equal(ia, want.idx, err_msg=f"{what}: model idx")
            np.testing.assert_array_equal(xa, want.act, err_msg=f"{what}: model act")
        self.columns(what)
        return ia, xa, sa

    def run_ticks(self, T, k, mode, seed):
        ra, rb = self.a.run_ticks(T, k, mode, seed), self.b.run_ticks(T, k, mode, seed)
        np.testing.assert_array_equal(ra, rb, err_msg=str((self.where, "run_ticks", T, mode)))
        if self.m is not None:
            want = self.m.run_ticks(T, k, mode, seed)
            assert [dict(zip(ra.dtype.names, [int(v) for v in r])) for r in ra] == want, self.where
        self.columns((self.where, "run_ticks"))


def _records(am, rng, n, T, tz_ids):
    """upsert records: the adversarial population in the library's own domain"""
    return am.columns_to_records(population(rng, n, T, True, tz_ids))


def _walk(am, zmap, seed, n, model, steps=40):
    rng = np.random.default_rng(seed)
    tz_ids = zmap.ids_of(zones_usable(T0 - 86400, T0 + 86400))
    w = Twins(am, zmap, n, model=model, seed=seed)
    T = T0
    hold = False
    reached = set()
    try:
        cols = population(rng, n, T, model is False, tz_ids)
        w.both("load_range", 0, cols)
        w.model("load", 0, cols)
        for step in range(steps):
            calls = ["upsert", "remove", "post", "post", "load", "tick", "tick", "tick", "tick", "run_ticks", "hold"]
            if not model:
                calls += ["spec", "spec", "restore"]
            call = calls[rng.integers(len(calls))]
            w.where = (seed, step, call)
            k = int(rng.integers(1, max(2, n // 8)))
            slots = rng.integers(0, n, k).astype(np.uint64)
            if call == "upsert":
                recs = _records(am, rng, k, T, tz_ids)
                w.both("upsert", slots, recs)
                w.model("upsert", slots, recs)
            elif call == "spec":  # ras (and the rest of the spec) edited, the status kept
                recs = am.columns_to_records(w.a.read(slots))
                recs["ras"] = rng.choice([1, 5, 60, 3600, 86400], k).astype(np.int32)
                w.both("update_spec", slots, recs)
            elif call == "remove":
                w.both("remove", slots)
                w.model("remove", slots)
            elif call == "post":
                if rng.integers(2):  # dense: applied inside the sweep rather than by the drain
                    slots = np.arange(n, dtype=np.uint64)
                    k = n
                phase = rng.integers(0, 3, k).astype(np.uint8)
                rphase = rng.integers(0, 3, k).astype(np.uint8)
                w.both("post_result", slots, phase, rphase)
                w.model("post", slots, phase, rphase)
            elif call == "load":
                first = int(rng.integers(0, n))
                part = population(rng, int(rng.integers(1, n - first + 1)), T, model is False, tz_ids)
                w.both("load_range", first, part)
                w.model("load", first, part)
            elif call == "restore":  # a checkpoint, calls staged over it, then the checkpoint restored
                blob = [w.a.checkpoint(), w.b.checkpoint()]
                recs = _records(am, rng, k, T, tz_ids)
                w.both("upsert", slots, recs)
                w.a.restore(blob[0])
                w.b.restore(blob[1])
                w.columns(w.where)
            elif call == "hold":
                hold = not hold
                w.both("set_hold_in_flight", hold)
                w.model("set_hold", hold)
                reached.add(("hold", hold))
            elif call == "run_ticks":
                if hold:  # (refused with the hold on)
                    continue
                mode = int(rng.choice([0, FULL, CLOSED, BLOCKED, BLOCKED | CLOSED]))
                w.run_ticks(T + 1, 3, mode, seed)
                T += 3
                reached.add(("run_ticks", mode))
            else:
                T += int(rng.choice([0, 1, 59, 60, -1, 3600, 86399]))
                mode = int(rng.choice([0, 0, 0, FULL, CLOSED]))
                if hold and w.m is not None:
                    mode &= ~CLOSED
                entry = str(rng.choice(["tick", "tick_view", "tick_device"]))
                try:
                    w.tick(T, mode, entry)
                except am.AmError as e:  # closed loop with the hold on: refused by both
                    assert e.code == am.AM_E_INVAL and (mode & CLOSED), e
                    with pytest.raises(am.AmError):
                        getattr(w.b, entry)(T, mode=mode) if entry != "tick_device" else w.dev[1].tick(am, w.b, T, mode)
                    continue
                reached.add(("tick", mode))
        w.where = (seed, "end")  # a closed-loop tick and the plain tick after it, in every walk
        w.both("set_hold_in_flight", False)
        w.model("set_hold", False)
        w.tick(T + 1, CLOSED)
        w.tick(T + 2)
        return reached
    finally:
        w.close()


@pytest.mark.parametrize("k,seed,n,model", [(0, 1, 1025, True), (1, 2, 3001, True), (2, 3, 1025, False),
                                            (3, 4, 4099, False), (4, 5, 257, True)])
def test_twin_walks(am, zmap, k, seed, n, model):
    reached = _walk(am, zmap, seed, _capacity(k, n), model)
    assert ("tick", 0) in reached, reached


# ---- the epoch window and the words' edges ----------------------------------------------------------------------
def _interval_cols(am, rows):
    """columns of interval records: rows of (ras, finished_at, armed, phase flags)"""
    recs = []
    for ras, fa, armed, extra in rows:
        rc, r = am.classify(repeat_after_sec=max(ras, 1), finished_at=fa, timer_armed=armed)
        assert rc == 0
        r["ras"] = ras
        r["flags"] |= np.uint32(extra)
        recs.append(r)
    return am.records_to_columns(np.concatenate(recs))


def test_epoch_window_edges_and_clamped_words(am, zmap):
    """ticks at E, E + 2^32 - 2, E + 2^32 - 1 and E - 1 (both outside the window: the words are rebuilt at a new
    epoch) and back, over records whose words are 0, clamped to 0xFFFFFFFF, and on either side of each tick"""
    E = T0 - LEAD
    edges = [E, E + SPAN - 1, E + SPAN, E - 1, T0, E + SPAN - 1]
    rows = [(60, T0 - 60, True, 0), (60, T0, True, 0), (3600, -(1 << 40), True, 0), ((1 << 31) - 1, 1 << 40, True, 0),
            (1, T0 + (1 << 33), True, 0), (5, T0 + 5, False, 0)]
    for t in edges:  # due exactly at, one second after and one second before each edge
        for d in (-1, 0, 1):
            rows.append((60, t + d - 60, True, 0))
            rows.append(((1 << 31) - 1, t + d - ((1 << 31) - 1), True, 0))
    cols = _interval_cols(am, rows)
    n = len(cols["flags"])
    w = Twins(am, zmap, n)
    try:
        w.both("load_range", 0, cols)
        w.model("load", 0, cols)
        w.where = "build"
        w.tick(T0)
        for t in edges:
            w.where = ("edge", t - E)
            w.tick(t)
            w.tick(t, FULL)
    finally:
        w.close()


def test_posted_phases_stopped_and_unarmed(am, zmap):
    """posted phases with ras <= 0 and > 0 (through the drain and, dense, through the sweep), unarmed timers whatever
    the word says, STOPPED reported with a result in the same tick, then the ticks after"""
    rng = np.random.default_rng(7)
    n = 2048
    cols = population(rng, n, T0, False, [])  # (ras 0, -1 and INT32_MIN on interval kinds too)
    w = Twins(am, zmap, n)
    try:
        w.both("load_range", 0, cols)
        w.model("load", 0, cols)
        w.where = "loaded"
        w.tick(T0)
        for t, dense in ((T0 + 1, False), (T0 + 60, True), (T0 + 61, False)):
            k = n if dense else 40
            slots = rng.choice(n, k, replace=False).astype(np.uint64)
            phase = rng.integers(0, 3, k).astype(np.uint8)
            rphase = rng.integers(0, 3, k).astype(np.uint8)
            w.both("post_result", slots, phase, rphase)
            w.model("post", slots, phase, rphase)
            w.where = ("posted", t, dense)
            w.tick(t)
        # STOPPED not yet reported, with a posted phase: both set finishedAt = T in one tick
        stop = w.a.read_range(0, n)
        kinds = stop["flags"] & np.uint32(am.KIND_MASK)
        sel = np.flatnonzero(kinds == am.KIND_STOPPED)[:30].astype(np.uint64)
        assert len(sel)
        stopped = {k: v[sel.astype(np.int64)].copy() for k, v in stop.items()}
        stopped["flags"] &= np.uint32(~am.F_STOPPED_REPORTED & 0xFFFFFFFF)
        for first, s in enumerate(sel.tolist()):
            one = {k: v[first:first + 1].copy() for k, v in stopped.items()}
            w.both("load_range", s, one)
            w.model("load", s, one)
        w.both("post_result", sel, np.ones(len(sel), np.uint8))
        w.model("post", sel, np.ones(len(sel), np.uint8))
        w.where = "stopped with a result"
        w.tick(T0 + 120)
        w.tick(T0 + 121)
    finally:
        w.close()


def test_spec_edit_restore_and_delta_restore(am, zmap):
    """a spec edit of ras between two ticks, a restore and a delta restore each followed by a tick: the restored
    handles (words, and finished_at handed out) tick as the producer does"""
    rng = np.random.default_rng(11)
    n = 3001
    cols = population(rng, n, T0, True, [])
    p = am.Sweep(capacity=n)  # the producer of the chain
    w = Twins(am, zmap, n, model=False)
    try:
        for s in (p, w.a, w.b):
            s.load_range(0, cols)
            s.tick(T0)
        w.where = "spec"
        slots = rng.choice(n, 200, replace=False).astype(np.uint64)
        recs = am.columns_to_records(w.a.read(slots))
        recs["ras"] = rng.choice([1, 30, 7200], len(slots)).astype(np.int32)
        for s in (p, w.a, w.b):
            s.update_spec(slots, recs)
        w.tick(T0 + 30)
        p.tick(T0 + 30)
        root = p.checkpoint_chain()
        w.both("restore", root)
        w.columns("restored")
        # the producer moves on: results, an upsert and one tick; the restorers apply the delta and tick with it
        post = rng.choice(n, 300, replace=False).astype(np.uint64)
        p.post_result(post, np.ones(len(post), np.uint8))
        p.upsert(slots[:10], _records(am, rng, 10, T0, []))
        p.tick(T0 + 31)
        delta, changed = p.checkpoint_delta()
        assert changed > 0
        w.both("restore_delta", delta)
        want = p.tick(T0 + 95)
        w.where = "delta restored"
        got = w.tick(T0 + 95)
        assert want[2] == got[2]
        np.testing.assert_array_equal(want[0], got[0])
        np.testing.assert_array_equal(want[1], got[1])
        pc = p.read_range(0, n)
        ac = w.a.read_range(0, n)
        for name in am.COLUMN_NAMES:
            np.testing.assert_array_equal(pc[name], ac[name], err_msg=name)
    finally:
        p.close()
        w.close()


def test_a_write_through_the_pointer_is_seen_by_the_next_tick(am, zmap):
    """a handle that has built its words and then hands out finished_at: the caller's write decides the next tick"""
    rng = np.random.default_rng(13)
    n = 1025
    cols = _interval_cols(am, [(60, T0 - 30, True, 0)] * n)
    w = Twins(am, zmap, n)
    try:
        w.both("load_range", 0, cols)
        w.model("load", 0, cols)
        w.where = "built"
        assert len(w.tick(T0)[0]) == 0
        slots = rng.choice(n, 100, replace=False)
        for s in (w.a, w.b):
            _write_column(am, s, "finished_at", slots, np.full(len(slots), T0 - 100))
        w.m.c["finished_at"][slots] = T0 - 100
        w.where = "written"
        idx = w.tick(T0 + 1)[0]
        np.testing.assert_array_equal(idx, np.sort(slots).astype(np.uint64))
    finally:
        w.close()
