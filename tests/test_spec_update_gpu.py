"""Spec updates (am_sweep_update_spec, DESIGN §6 item 20): the hand-derived cases (tests/spec_update_cases.py) and
random call sequences through every tick entry point against tests/spec_update_model.py (the handle model with the
submit budget and spec updates), compared after every tick by tests/handle_pair.py — list, statistics, the sixteen columns, in_flight, the
timed-out lists, the changes and their details, the waits; every order of an upsert, a spec update, a posted phase and
a remove of one slot within one drain; a status echo against an upsert of the same stale status, also after a restore;
run_ticks, simulate and checkpoints draining staged spec updates; the refusals; the launch counts; and, on an H100, a
10 M-record spec refresh of config 2 followed by a tick against the oracle."""
import itertools
import zlib

import numpy as np
import pytest

import admission_oracle as ao
import amgen
import hold_oracle
import spec_update_cases
from adversarial import ZoneMap, population, zones_usable
from handle_pair import Pair, emulated
from spec_update_model import SpecModel
from timeout_cases import M0, rec

pytestmark = pytest.mark.gpu

DAY, HOUR = 86400, 3600
T_OCT = 1790812800  # 2026-10-01 00:00:00 UTC
FULL, CATCH = 0x2, 0x8
NONE = hold_oracle.NOT_IN_FLIGHT
ENTRIES = ["tick", "tick_short", "tick_view", "tick_device", "tick_shard"]


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


class SpecPair(Pair):
    """tests/handle_pair.py's Pair with update_spec on both sides, SpecModel as the model (the waits and the last
    admission compared after every tick) and a restart through a checkpoint.  `every_slot` as in Pair."""

    def __init__(self, am, zmap, n, hold=False, remedy=False, track=False, details=False, entry="tick", cap=1,
                 every_slot=True):
        self.am, self.entry, self.cap, self.every_slot = am, entry, cap, every_slot
        self.n = n
        self.s = am.Sweep(capacity=n)
        self.m = SpecModel(zmap, n)
        for on, switch in ((hold, self.set_hold), (remedy, self.set_remedy), (track, self.set_track),
                           (details, self.set_details)):
            if on:
                switch(True)
        self.dev = None
        self.timed_total = self.rtimed_total = self.started = self.listed = self.detailed = 0

    def update_spec(self, slots, recs):
        self.s.update_spec(slots, recs)
        self.m.update_spec(slots, recs)

    # the handle's queries drain what is staged
    def cols(self):
        self.m.drained()
        return super().cols()

    def in_flight(self):
        self.m.drained()
        return super().in_flight()

    def remedy_in_flight(self):
        self.m.drained()
        return super().remedy_in_flight()

    def deferred(self):
        self.m.drained()
        return self.s.deferred(0, self.n)

    def set_budget(self, v):
        self._switch(self.s.set_submit_budget, self.m.set_budget, v)

    def restart(self):
        """a checkpoint of the handle (it drains what is staged) restored into a fresh one with the same switches and
        budget, which carries on"""
        am, m = self.am, self.m
        blob = self.s.checkpoint()
        m.drained()
        sw = am.checkpoint_info(blob)["switches"]
        t = am.Sweep(capacity=self.n)
        for bit, call in ((am.CKPT_HOLD, t.set_hold_in_flight), (am.CKPT_REMEDY, t.set_hold_remedy),
                          (am.CKPT_TRACK, t.set_track_changes), (am.CKPT_DETAILS, t.set_change_details)):
            if sw & bit:
                call(True)
        if m.adm and m.hold:
            t.set_submit_budget(0)
            t.set_submit_budget(None if m.budget == ao.UNLIMITED else m.budget)
        t.restore(blob)
        self.s.close()
        self.s, self.dev = t, None

    def tick(self, T, mode=0, entry=None):
        got = super().tick(T, mode, entry)
        np.testing.assert_array_equal(self.s.deferred(0, self.n), self.m.deferred(0, self.n), err_msg=f"{T}: deferred")
        if self.m.adm:
            assert self.s.last_admission() == self.m.last_admission(), T
        return got


def _echo_of(am, m, slots):
    """the records a controller builds from its CRs when their status is the model's: a spec update of them is a
    status echo with an unchanged spec"""
    recs = am.columns_to_records({k: v[slots] for k, v in m.cols().items()})
    recs["wf_timeout"] = m.wf[slots]
    return recs


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("case", spec_update_cases.CASES, ids=lambda c: c.__name__)
def test_hand_derived_cases(am, zmap, case, entry):
    p = SpecPair(am, zmap, 8, hold=True, remedy=True, track=True, details=True, entry=entry)
    try:
        case(am, p)
    finally:
        p.close()


SEQ = "USPX"  # upsert, spec update, posted phase (workflow and remedy), remove


@pytest.mark.parametrize("switches", ["plain", "hold", "all"])
def test_every_order_within_one_drain(am, zmap, switches):
    """slot j gets the j-th sequence of one to three calls out of U, S, P, X (84 slots), interleaved across slots in
    one drain; the tick and the one after it equal the model's"""
    seqs = [s for k in (1, 2, 3) for s in itertools.product(SEQ, repeat=k)]
    n = len(seqs) + 4
    rng = np.random.default_rng(len(switches))
    hold, full = switches != "plain", switches == "all"
    p = SpecPair(am, zmap, n, hold=hold, remedy=full, track=full, details=full, every_slot=False)
    T = M0 + 3
    base = [rec(am, 40 if hold else 0, repeat_after_sec=30, finished_at=T - 100, has_remedy=True,
                remedy_runs_limit=2, success_count=3, failed_count=1)] * n
    p.upsert(np.arange(n), np.concatenate(base))
    try:
        p.tick(T)  # every check submitted (held with the hold)
        specs = [rec(am, 15, cron="*/2 * * * *", has_remedy=True, remedy_runs_limit=5),
                 rec(am, 0, repeat_after_sec=7, remedy_runs_limit=1), rec(am, 0)]
        queue = [[(c, j) for c in s] for j, s in enumerate(seqs)]
        while any(queue):  # round-robin with random picks: per slot in sequence order
            j = int(rng.choice([j for j, q in enumerate(queue) if q]))
            c, slot = queue[j].pop(0)
            if c == "U":
                p.upsert([slot], rec(am, 20, repeat_after_sec=11, finished_at=T - 5, success_count=9))
            elif c == "S":
                p.update_spec([slot], specs[int(rng.integers(0, len(specs)))])
            elif c == "P":
                p.post([slot], [int(rng.integers(1, 3))], [int(rng.integers(0, 3))])
            else:
                p.remove([slot])
        p.tick(T + 17)
        p.tick(T + 60)
    finally:
        p.close()


STEPS = [1, 1, 59, 1, 1, 60, 1, 2, 1, 57, 1, 0, 1, -30, 1, 600, 1, 1, 60, 1, 1, 59, 1, 1]
CONFIGS = ["plain", "hold", "timeouts_remedy_budget", "catch_up_details", "full_scan_track"]


@pytest.mark.parametrize("config", CONFIGS)
@pytest.mark.parametrize("entry", ENTRIES)
def test_random_call_sequences_equal_the_model(am, zmap, entry, config):
    """spec updates (new specs and status echoes), upserts, removes, posts, loads and reads between ticks, a restart
    through a checkpoint with calls staged, and without the hold runs of ticks"""
    n = 1500
    rng = np.random.default_rng(zlib.crc32(f"spec {entry} {config}".encode()))
    T = T_OCT + 9 * DAY + 11 * HOUR - 2
    hold = config != "plain"
    details = "details" in config
    mode = CATCH if "catch_up" in config else FULL if "full_scan" in config else 0
    wf = "timeouts" in config
    zones = zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))
    p = SpecPair(am, zmap, n, hold=hold, remedy=hold and ("remedy" in config or details),
                 track=details or "track" in config, details=details, entry=entry, cap=5, every_slot=False)

    def records(k):
        recs = am.columns_to_records(population(rng, k, T, True, zones))
        recs["wf_timeout"] = rng.integers(0, 200, k) if wf else 0
        return recs

    counts = dict.fromkeys(("spec", "echo", "ran"), 0)
    try:
        p.upsert(np.arange(n), records(n))
        for k, step in enumerate(STEPS):
            if "budget" in config and k % 4 == 0:
                p.set_budget([0, 7, 40, 300, None][int(rng.integers(0, 5))] if k else 50)
            for _ in range(int(rng.integers(1, 5))):
                r = rng.random()
                sl = rng.choice(n, int(rng.integers(1, 80)))  # (duplicates: the latest entry of a slot wins)
                if r < 0.3:
                    p.update_spec(sl, records(len(sl)))
                    counts["spec"] += len(sl)
                elif r < 0.45:
                    p.update_spec(sl, _echo_of(am, p.m, sl))
                    counts["echo"] += len(sl)
                elif r < 0.6:
                    p.upsert(sl, records(len(sl)))
                elif r < 0.7:
                    p.remove(sl[:10])
                elif r < 0.9:
                    busy = np.flatnonzero(p.m.since != NONE)
                    ps = np.concatenate([rng.choice(busy, min(len(busy), 40), replace=False), sl[:10]])
                    p.post(ps, rng.integers(0, 3, len(ps)), rng.integers(0, 3, len(ps)).astype(np.uint8))
                elif r < 0.95:
                    p.load(int(rng.integers(0, n - 50)), population(rng, 50, T, True, zones))
                else:
                    p.read(sl)
            if k in (7, 16):
                p.update_spec(rng.choice(n, 30), records(30))  # staged into the checkpoint's drain
                p.restart()
            if not hold and k % 6 == 5:
                want = p.m.run_ticks(T + 1, 3)
                got = p.s.run_ticks(T + 1, 3)
                for j in range(3):
                    assert {f: int(got[j][f]) for f in am.abi.STAT_FIELDS} == want[j], (k, j)
                T += 3
                counts["ran"] += 1
                continue
            T += step
            p.tick(T, mode)
        assert counts["spec"] > 100 and counts["echo"] > 50, counts
    finally:
        p.close()


def test_simulate_drains_spec_updates(am, zmap):
    """am_sweep_simulate drains staged spec updates as a tick does: a check whose interval the update shortens is
    submitted by the simulation's first tick"""
    with am.Sweep(capacity=4) as s:
        s.set_hold_in_flight(True)
        s.set_hold_remedy(True)
        s.upsert([0], rec(am, 0, repeat_after_sec=600, finished_at=M0 - 10))
        s.tick(M0)
        s.update_spec([0], rec(am, 0, repeat_after_sec=5))
        rows, _ = s.simulate(M0 + 1, 1, 0, 1, (100, 100, 100, 100))
        assert int(rows[0]["n_submit_hc"]) == 1


def _stale_restore(am, via):
    """a check counted up to S = 5 is checkpointed; a restarted controller restores the blob, then re-applies its CR
    from etcd's older status (S = 3, finishedAt 1000 s ago) through `via`; the next tick"""
    with am.Sweep(capacity=4) as s:
        s.set_hold_in_flight(True)
        s.upsert([0], rec(am, 0, repeat_after_sec=60, finished_at=M0 - 100, success_count=4))
        s.tick(M0)
        s.post_result([0], [1])
        s.tick(M0 + 5)
        blob = s.checkpoint()
    with am.Sweep(capacity=4) as t:
        t.set_hold_in_flight(True)
        t.restore(blob)
        getattr(t, via)([0], rec(am, 0, repeat_after_sec=60, finished_at=M0 - 1000, success_count=3))
        idx, act, _ = t.tick(M0 + 6)
        return idx, act, t.read_range(0, 1)


def test_stale_status_after_a_restore(am):
    idx, act, c = _stale_restore(am, "upsert")
    assert c["success"][0] == 3 and list(idx) == [0]  # rolled back, and resubmitted at once
    idx, act, c = _stale_restore(am, "update_spec")
    assert c["success"][0] == 5 and c["finished_at"][0] == M0 + 5 and len(idx) == 0


def test_refusals_stage_nothing(am, zmap):
    with am.Sweep(capacity=8) as s:
        s.upsert([0], rec(am, 0, repeat_after_sec=60, finished_at=M0))
        before = s.read_range(0, 8)
        bad_zone = rec(am, 0, cron="0 9 * * *")
        bad_zone["flags"] |= np.uint32(255 << 24)
        for recs, slots, code in ((bad_zone, [0], am.AM_E_INVAL), (rec(am, -1, repeat_after_sec=5), [0], am.AM_E_RANGE),
                                  (rec(am, 0, repeat_after_sec=5), [8], am.AM_E_RANGE)):
            with pytest.raises(am.AmError) as e:
                s.update_spec(slots, recs)
            assert e.value.code == code
        lib = s._lib
        r = rec(am, 0, repeat_after_sec=5)
        idx = np.zeros(1, np.uint64)
        assert lib.am_sweep_update_spec(None, 1, idx.ctypes.data, r.ctypes.data) == am.AM_E_INVAL
        assert lib.am_sweep_update_spec(s._h, 1, None, r.ctypes.data) == am.AM_E_INVAL
        assert lib.am_sweep_update_spec(s._h, 1, idx.ctypes.data, None) == am.AM_E_INVAL
        assert lib.am_sweep_update_spec(s._h, 0, None, None) == am.AM_OK
        after = s.read_range(0, 8)
        for name in am.COLUMN_NAMES:
            np.testing.assert_array_equal(after[name], before[name], err_msg=name)


def test_launch_counts(am, zmap):
    """a drain with spec updates launches the apply pass (one kernel) on top of what the same drain without them
    launches; once a drain has none, the handle launches what a handle that never staged one does"""
    n = 4096
    rng = np.random.default_rng(4)
    T = T_OCT + 3 * HOUR
    cols = population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY)))
    with am.Sweep(capacity=n) as a, am.Sweep(capacity=n) as b:
        per = {id(a): [], id(b): []}
        for s in (a, b):
            s.set_hold_in_flight(True)
            s.set_track_changes(True)
            s.load_range(0, cols)
        recs = am.columns_to_records({k: v[:64] for k, v in cols.items()})
        for t in range(4):
            for s in (a, b):
                l0 = s.launch_count
                s.upsert(np.arange(64), recs)
                s.post_result(np.arange(100, n, 9), np.full(len(range(100, n, 9)), 1, np.uint8))
                if s is b:
                    s.update_spec(np.arange(64, 128), am.columns_to_records({k: v[64:128] for k, v in cols.items()}))
                s.tick(T + 60 * t)
                per[id(s)].append(s.launch_count - l0)
        assert [y - x for x, y in zip(per[id(a)], per[id(b)])] == [1] * 4, per
        for s in (a, b):  # a drain without spec updates: the same kernels again
            l0 = s.launch_count
            s.upsert(np.arange(64), recs)
            s.tick(T + 600)
            per[id(s)].append(s.launch_count - l0)
        assert per[id(a)][-1] == per[id(b)][-1], per


def test_full_size(am, zmap):
    """config 2 at 10 M records: a tick, a spec refresh of every record from another seed's population (kinds, masks
    and zones change; the status is the handle's), a tick; the list, statistics and columns against the oracle run on
    the refreshed columns"""
    if emulated(am):
        pytest.skip("10 M records: the GPU")
    n, T0 = 10_000_000, amgen.T0_MON_0915
    classify = am.load().am_healthcheck_classify
    cols = amgen.fill(2, 2, 0, n, T0 - 30, classify)
    spec = am.columns_to_records(amgen.fill(2, 3, 0, n, T0 - 30, classify))
    m = SpecModel(zmap, n)
    with am.Sweep(capacity=n) as s:
        s.load_range(0, cols)
        s.tick(T0 - 1)
        m.c = s.read_range(0, n)
        m.hwm = n
        s.update_spec(np.arange(n, dtype=np.uint64), spec)
        m.update_spec(np.arange(n), spec)
        idx, act, st = s.tick(T0)
        want_idx, want_act, want_st = zmap.sweep(m.c, T0)
        assert st == want_st
        np.testing.assert_array_equal(idx, want_idx)
        np.testing.assert_array_equal(act, want_act)
        dev = s.read_range(0, n)
        for name in am.COLUMN_NAMES:
            np.testing.assert_array_equal(dev[name], m.c[name], err_msg=name)
