"""Submit budget (am_sweep_set_submit_budget): every tick entry point against tests/admission_model.py — list,
statistics, the sixteen columns, in_flight, both timed-out lists (tests/handle_pair.py), and after every tick
am_sweep_deferred and am_sweep_last_admission — with the budget changed between ticks; the no-starvation bound; the
refusals; launch counts without a budget; checkpoints taken mid-backlog, restored into one handle and into two
resharded ones; am_sweep_simulate tick by tick against tests/sim_driver.py's loop on the model; and, on an H100, config 2
at 10 M records against an unlimited handle."""
import zlib

import numpy as np
import pytest

import amgen
import admission_cases
import admission_oracle as ao
import hold_oracle
from adversarial import ZoneMap, population, zones_usable
from admission_model import AdmissionModel
from handle_model import Refused
from handle_pair import Pair, emulated
import sim_driver

pytestmark = pytest.mark.gpu

DAY, HOUR = 86400, 3600
T_OCT = 1790812800  # 2026-10-01 00:00:00 UTC
FULL, CATCH = 0x2, 0x8
NONE = hold_oracle.NOT_IN_FLIGHT


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


class AdmPair(Pair):
    """tests/handle_pair.py's Pair with AdmissionModel as the model and the admission compared after every tick"""

    def __init__(self, am, zmap, n_or_cols, hold=True, remedy=False, entry="tick", cap=1, track=False, details=False):
        cols = None if isinstance(n_or_cols, int) else n_or_cols
        self.am, self.entry, self.cap, self.every_slot = am, entry, cap, True
        self.n = n_or_cols if cols is None else len(cols["flags"])
        self.s = am.Sweep(capacity=self.n)
        self.m = AdmissionModel(zmap, self.n)
        self.set_hold(hold)
        if remedy:
            self.set_remedy(True)
        if track:
            self.set_track(True)
        if details:
            self.set_details(True)
        if cols is not None:
            self.load(0, cols)
        self.dev = None
        self.timed_total = self.rtimed_total = self.started = self.listed = self.detailed = 0

    def set_budget(self, v):
        self._switch(self.s.set_submit_budget, self.m.set_budget, v)

    def deferred(self):
        return self.s.deferred(0, self.n)

    def last_admission(self):
        return self.s.last_admission()

    def tick(self, T, mode=0, entry=None):
        got = super().tick(T, mode, entry)
        np.testing.assert_array_equal(self.s.deferred(0, self.n), self.m.deferred(0, self.n), err_msg=f"{T}: deferred")
        if self.m.adm:
            assert self.s.last_admission() == self.m.last_admission(), (T, self.s.last_admission())
        return got


def _records(am, rng, n, T, zmap, wf=False):
    recs = am.columns_to_records(population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY))))
    if wf:
        recs["wf_timeout"] = rng.integers(0, 200, n)
    return recs


STEPS = [1, 1, 59, 1, 1, 60, 1, 2, 1, 57, 1, 0, 1, -30, 1, 600, 1, 1, 60, 1, 1, 59, 1, 1]
BUDGETS = [0, 1, 7, 40, 300, None]


@pytest.mark.parametrize("config", ["hold", "timeouts_remedy", "catch_up", "full_scan_details"])
@pytest.mark.parametrize("entry", ["tick", "tick_short", "tick_view", "tick_device", "tick_shard"])
def test_budgeted_ticks_equal_the_model(am, zmap, entry, config):
    n = 2500
    rng = np.random.default_rng(zlib.crc32(f"{entry} {config}".encode()))
    T = T_OCT + 9 * DAY + 11 * HOUR - 2
    mode = {"catch_up": CATCH, "full_scan_details": FULL}.get(config, 0)
    wf = config == "timeouts_remedy"
    det = config == "full_scan_details"  # (status changes and their details under a budget)
    p = AdmPair(am, zmap, population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))),
                remedy=wf or det, entry=entry, cap=5, track=det, details=det)
    deferred_seen = ended = 0
    try:
        if wf:
            p.upsert(np.arange(n), _records(am, rng, n, T, zmap, wf=True))
        for k, step in enumerate(STEPS):
            if k % 3 == 0:
                p.set_budget(BUDGETS[int(rng.integers(0, len(BUDGETS)))] if k else 50)
            if k:
                r = rng.random()
                waiting = np.flatnonzero(p.m.wait != ao.NOT_WAITING)
                if r < 0.25:
                    sl = rng.choice(n, 30, replace=False)
                    if len(waiting):  # an upsert keeps the wait
                        sl = np.unique(np.concatenate([sl, waiting[:10]]))
                    p.upsert(sl, _records(am, rng, len(sl), T, zmap, wf=wf))
                elif r < 0.4:
                    p.remove(np.concatenate([rng.choice(n, 10, replace=False), waiting[:5]]))
                    ended += min(len(waiting), 5)
                elif r < 0.5:
                    p.load(int(rng.integers(0, n - 100)), population(rng, 100, T, True,
                                                                     zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))))
                busy = np.flatnonzero(p.m.since != NONE)
                sl = np.concatenate([rng.choice(busy, min(len(busy), 60), replace=False), waiting[5:10]])
                if len(sl):
                    p.post(sl, rng.integers(1, 3, len(sl)), rng.integers(0, 3, len(sl)).astype(np.uint8))
                if len(waiting) > 10:  # a remedy phase alone keeps the wait
                    p.post(waiting[10:15], np.zeros(len(waiting[10:15]), np.uint8),
                           rng.integers(1, 3, len(waiting[10:15])).astype(np.uint8))
            T += step
            p.tick(T, mode)
            deferred_seen += int((p.m.wait != ao.NOT_WAITING).sum())
        assert deferred_seen > 500, deferred_seen
    finally:
        p.close()


@pytest.mark.parametrize("entry", ["tick", "tick_short", "tick_view", "tick_device", "tick_shard"])
@pytest.mark.parametrize("case", admission_cases.CASES, ids=lambda c: c.__name__)
def test_hand_derived_cases(am, zmap, case, entry):
    p = AdmPair(am, zmap, 8, remedy=True, entry=entry)
    try:
        case(am, p)
    finally:
        p.close()


def test_no_starvation_and_order(am, zmap):
    """a waiting check is admitted within ceil(ahead / budget) ticks; admissions come out in (second, index) order"""
    n, B = 3000, 37
    rng = np.random.default_rng(5)
    T = T_OCT + 3 * DAY + 7
    cols = population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY)))
    p = AdmPair(am, zmap, cols)
    try:
        p.set_budget(B)
        bound = {}
        for t in range(40):
            before = p.m.wait.copy()
            got = p.tick(T + t)
            sub = got.idx[(got.act & 1) != 0].astype(np.int64)
            assert len(sub) <= B
            w = np.flatnonzero(before != ao.NOT_WAITING)
            order = w[np.lexsort((w, before[w]))]
            for r, i in enumerate(order):  # the admission bound of every slot that waited before this tick
                bound.setdefault(int(i), t + r // B)
            for i in sub:
                bound.pop(int(i), None)
            assert all(v > t for i, v in bound.items() if p.m.wait[i] != ao.NOT_WAITING), t
    finally:
        p.close()


def test_refusals(am, zmap):
    n = 512
    rng = np.random.default_rng(9)
    T = T_OCT + 60 * 17
    cols = population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY)))
    with am.Sweep(capacity=n) as s:
        with pytest.raises(am.AmError) as e:
            s.set_submit_budget(10)  # hold off
        assert e.value.code == am.AM_E_INVAL
        s.set_hold_in_flight(True)
        with pytest.raises(am.AmError) as e:
            s.last_admission()  # no admission state yet
        assert e.value.code == am.AM_E_INVAL
        s.set_hold_remedy(True)
        s.load_range(0, cols)
        s.set_submit_budget(3)
        s.tick(T)
        adm = s.last_admission()
        assert adm["n_admitted"] == 3 and adm["n_deferred"] > 0 and adm["oldest_deferred"] == T
        assert s.next_due(T + 1) == T + 2  # a waiting check is due at the next second
        P = T
        for budget in (3, None):  # the blocked run has no admission: refused under a budget and while checks wait
            s.set_submit_budget(budget)
            with pytest.raises(am.AmError) as e:
                s.simulate(T + 1, 5, mode=0x4)
            assert e.value.code == am.AM_E_INVAL
        s.set_submit_budget(3)
        s.tick(P + 1)  # nothing happened: the next tick goes on from the backlog
        assert s.last_admission()["n_admitted"] == 3
        assert am.checkpoint_info(s.checkpoint())["switches"] & am.CKPT_ADMISSION  # a blob carries the waits
        s.set_submit_budget(None)
        s.remove(np.flatnonzero(s.deferred(0, n) != ao.NOT_WAITING))
        assert (s.deferred(0, n) == ao.NOT_WAITING).all()  # (drained: no check waits, the FIFO still has entries)
        s.simulate(P + 2, 3, mode=0x4)
        s.set_hold_in_flight(False)  # resets everything
        s.set_hold_in_flight(True)
        assert s.last_admission() == ao.empty_admission()
        assert (s.deferred(0, n) == ao.NOT_WAITING).all()


def test_launch_counts(am, zmap):
    """a handle that never sets a budget launches what it launched before; one with the admission state adds six
    kernels per tick and one per drain"""
    n = 2048
    rng = np.random.default_rng(3)
    T = T_OCT + 3 * HOUR
    cols = population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY)))
    with am.Sweep(capacity=n) as a, am.Sweep(capacity=n) as b, am.Sweep(capacity=n) as c:
        for s in (a, b, c):
            s.set_hold_in_flight(True)
            s.load_range(0, cols)
        b.set_submit_budget(None)  # unlimited: allocates nothing
        c.set_submit_budget(10 ** 9)
        per = {id(s): [] for s in (a, b, c)}
        for t in range(5):
            for s in (a, b, c):
                l0 = s.launch_count
                s.post_result(np.arange(0, n, 9), np.full(len(range(0, n, 9)), 1, np.uint8))
                s.tick(T + 60 * t)
                per[id(s)].append(s.launch_count - l0)
        assert per[id(a)] == per[id(b)], per
        assert [x - y for x, y in zip(per[id(c)], per[id(a)])] == [7] * 5, per


def test_model_refusals_match(am, zmap):
    m = AdmissionModel(zmap, 8)
    with pytest.raises(Refused):
        m.set_budget(1)
    m.set_hold(True)
    with pytest.raises(Refused):
        m.last_admission()


def _handle_like(am, src_info, capacity, shard_base=0):
    """a handle with a blob's switches, set as a controller sets them after am_checkpoint_info (a finite budget once
    for the admission state)"""
    t = am.Sweep(capacity=capacity, shard_base=shard_base)
    sw = src_info["switches"]
    for bit, call in ((am.CKPT_HOLD, t.set_hold_in_flight), (am.CKPT_REMEDY, t.set_hold_remedy),
                      (am.CKPT_TRACK, t.set_track_changes), (am.CKPT_DETAILS, t.set_change_details)):
        if sw & bit:
            call(True)
    if sw & am.CKPT_ADMISSION:
        t.set_submit_budget(0)
        t.set_submit_budget(None)
    return t


def _backlog(am, zmap, rng, n, T, wf):
    p = AdmPair(am, zmap, n, remedy=True, track=True)
    p.upsert(np.arange(n), _records(am, rng, n, T, zmap, wf=wf))
    p.set_budget(40)
    for k, step in enumerate([0, 1, 60, 1, 1, 59]):
        T += step
        if k == 3:
            busy = np.flatnonzero(p.m.since != NONE)[:50]
            p.post(busy, rng.integers(1, 3, len(busy)))
        p.tick(T)
    assert (p.m.wait != ao.NOT_WAITING).sum() > 300
    return p, T


@pytest.mark.parametrize("wf", [False, True], ids=["no_timeouts", "timeouts"])
def test_checkpoint_mid_backlog_one_handle(am, zmap, wf):
    """a blob taken mid-backlog carries every wait; restored into a fresh handle of the same shard, the handle goes on
    tick for tick as the model does (a restore is the identity on it)"""
    n = 3000
    rng = np.random.default_rng(21 + wf)
    p, T = _backlog(am, zmap, rng, n, T_OCT + 4 * DAY + 9 * HOUR + 30, wf)
    try:
        blob = p.s.checkpoint()
        info = am.checkpoint_info(blob)
        assert info["switches"] & am.CKPT_ADMISSION
        t = _handle_like(am, info, n)
        t.set_submit_budget(40)
        t.restore(blob)
        np.testing.assert_array_equal(t.deferred(0, n), p.m.deferred(0, n))
        p.s.close()
        p.s, p.dev = t, None
        for k, step in enumerate([1, 1, 58, 1, 2, 60, 1]):
            if k == 3:
                p.set_budget(int(rng.integers(0, 100)))
            T += step
            p.tick(T)
    finally:
        p.close()


def test_checkpoint_mid_backlog_resharded(am, zmap):
    """the blobs of one checkpoint cut at a new bound restore into two handles: their waits are the source's, and with
    the budget unlimited their next ticks together emit the source's list"""
    n, cut = 3000, 1337
    rng = np.random.default_rng(33)
    p, T = _backlog(am, zmap, rng, n, T_OCT + 6 * DAY + 30, True)
    shards = []
    try:
        for lo, hi in ((0, cut), (cut, n)):
            blob = p.s.checkpoint(lo, hi - lo)
            t = _handle_like(am, am.checkpoint_info(blob), hi - lo, shard_base=lo)
            t.restore(blob)
            shards.append(t)
        np.testing.assert_array_equal(np.concatenate([t.deferred(0, t.capacity) for t in shards]), p.m.deferred(0, n))
        p.set_budget(None)
        for t in shards:
            t.set_submit_budget(None)
        for step in (1, 1):
            T += step
            want = p.tick(T)
            got = [t.tick(T) for t in shards]
            np.testing.assert_array_equal(np.concatenate([g[0] for g in got]), want.idx)
            np.testing.assert_array_equal(np.concatenate([g[1] for g in got]), want.act)
            np.testing.assert_array_equal(np.concatenate([t.in_flight(0, t.capacity) for t in shards]), p.m.in_flight(0, n))
            assert all((t.deferred(0, t.capacity) == ao.NOT_WAITING).all() for t in shards)
    finally:
        for t in shards:
            t.close()
        p.close()


def test_simulate_tick_by_tick_honours_the_budget(am, zmap):
    """am_sweep_simulate under a budget is tests/sim_driver.py's loop of posts and ticks on the model: statistics and
    simulation rows per tick, then the columns, the runs in flight, the waits and the last admission"""
    n = 2000
    rng = np.random.default_rng(8)
    T = T_OCT + 2 * DAY + 5 * HOUR - 20
    params, seed = (2, 9, 3, 12), 77
    p = AdmPair(am, zmap, n, remedy=True)
    try:
        p.upsert(np.arange(n), _records(am, rng, n, T, zmap, wf=True))
        p.set_budget(25)
        p.tick(T)  # a backlog before the run
        T += 1
        for budget in (25, 0, 300, None):
            p.set_budget(budget)
            wrows, wsims = sim_driver.simulate(p.m, T, 30, 0, seed, params)
            rows, sims = p.s.simulate(T, 30, 0, seed, params)
            for k, (r, w) in enumerate(zip(rows, wrows)):
                gd = {f: int(r[f]) for f in am.abi.STAT_FIELDS}
                assert gd == w, (budget, k, {f: (gd[f], w[f]) for f in gd if gd[f] != w[f]})
            np.testing.assert_array_equal(np.array([tuple(x) for x in sims], dtype=np.int64).reshape(-1, 4),
                                          np.array(wsims, dtype=np.int64).reshape(-1, 4))
            dev = p.s.read_range(0, n)
            for name in am.COLUMN_NAMES:
                np.testing.assert_array_equal(dev[name], p.m.cols()[name], err_msg=f"{budget}: {name}")
            np.testing.assert_array_equal(p.s.in_flight(0, n), p.m.in_flight(0, n))
            np.testing.assert_array_equal(p.s.deferred(0, n), p.m.deferred(0, n))
            assert p.s.last_admission() == p.m.last_admission()
            T += 30
    finally:
        p.close()


@pytest.mark.parametrize("budget", [10_000, 1_000_000])
def test_full_size(am, budget):
    """config 2 at 10 M records, hold and workflow timeouts on, 120 consecutive ticks at a budget against a handle
    without one: at most `budget` submissions, min(budget, candidates) admitted, waiting checks before fresh ones and
    in (second, index) order, the counts of am_sweep_last_admission, and, once the backlog drains, the same runs in
    flight on both handles (every check either submitted is still held: nothing is posted)"""
    if emulated(am):
        pytest.skip("10 M records: the GPU")
    n, T0 = 10_000_000, amgen.T0_MON_0915
    cols = amgen.fill(2, 2, 0, n, T0 - 30, am.load().am_healthcheck_classify)
    with am.Sweep(capacity=n) as a, am.Sweep(capacity=n) as b:
        for s in (a, b):
            s.load_range(0, cols)
            s.set_hold_in_flight(True)
            rec = am.columns_to_records({k: v[:1] for k, v in cols.items()})
            rec["wf_timeout"] = 100000
            s.upsert([0], rec)
        b.set_submit_budget(budget)
        for k in range(120):
            T = T0 - 30 + k
            before = b.deferred(0, n)
            ia, aa, _ = a.tick_view(T)
            ib, ab, sb = b.tick_view(T)
            sub = ib[(ab & 1) != 0].astype(np.int64)
            adm = b.last_admission()
            assert len(sub) == sb["n_submit_hc"] == adm["n_admitted"] == min(budget, adm["n_candidates"]), (k, adm)
            if k == 0:  # the same state on both: the admitted are the first of the unlimited handle's submissions
                full = ia[(aa & 1) != 0].astype(np.int64)
                assert adm["n_candidates"] == len(full)
                np.testing.assert_array_equal(sub, full[:len(sub)])
            wait = b.deferred(0, n)
            waiting = wait != ao.NOT_WAITING
            assert adm["n_deferred"] == int(waiting.sum())
            assert adm["oldest_deferred"] == (int(wait[waiting].min()) if waiting.any() else ao.INT64_MAX)
            was = before[sub] != ao.NOT_WAITING
            old, fresh = sub[was], sub[~was]
            left = np.flatnonzero((before != ao.NOT_WAITING) & waiting)  # waited before and still waits
            if len(old) and len(left):  # admission order: (second, index)
                hi, lo = before[old].max(), before[left].min()
                assert (hi, old[before[old] == hi].max()) < (lo, left[before[left] == lo].min()), k
            if len(fresh):  # fresh ones only once no older check waits, and before the checks deferred now
                assert not len(left), k
                new = np.flatnonzero(wait == T)
                new = new[before[new] == ao.NOT_WAITING]
                assert not len(new) or fresh.max() < new.min(), k
        b.set_submit_budget(None)
        b.tick_view(T0 + 90)
        a.tick_view(T0 + 90)
        assert b.last_admission()["n_deferred"] == 0
        np.testing.assert_array_equal(a.in_flight(0, n) != NONE, b.in_flight(0, n) != NONE)
