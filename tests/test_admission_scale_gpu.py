"""The submit budget across admission groups (8192 records each) and at shard bases: a shard of 4 full groups, a partial
fifth group and a partial last tile, at base 0, at a base that is not a multiple of 32 and, for tick_device, past 2^32,
through every tick entry point, against tests/spec_update_model.py (the handle model with the budget and spec updates)
after every tick: list, statistics, columns, in_flight, the timed-out lists, the changes and their details, the waits
(deferred) and the last admission.  Each tick's budget is picked from a dry run of the model's candidate queue so that
the cut lands exactly on a group edge among the fresh candidates, one before it, one after it, inside the partial last
group, inside the waiting candidates, at 0, or past every candidate; the test asserts that every one of those cuts was made."""
import copy
import zlib
from collections import Counter

import numpy as np
import pytest

import admission_oracle as ao
import sim_driver
from adversarial import population, zones_usable
from handle_pair import emulated
from spec_update_model import SpecModel
from test_spec_update_gpu import NONE, SpecPair, zmap  # noqa: F401 (zmap: the module's fixture)
from timeout_cases import M0, rec

pytestmark = pytest.mark.gpu

GROUP = 8192  # records per admission group (kGroupRecords)
N = 4 * GROUP + 777
DAY = 86400
FULL, CATCH = 0x2, 0x8
STEPS = [1, 59, 1, 60, 1, 0, 1, -30, 1, 59, 1, 60, 1, 1, 58, 1]
CUTS = ["group_edge", "before_edge", "after_edge", "last_group", "waiting", "zero", "everyone"]


class ScalePair(SpecPair):
    """SpecPair (SpecModel, the waits and the last admission compared after every tick) on a handle at `shard_base`"""

    def __init__(self, am, zmap, n, shard_base, entry, switches=("hold", "remedy", "track", "details")):
        self.am, self.entry, self.cap, self.every_slot = am, entry, 5, False
        self.n = n
        self.s = am.Sweep(capacity=n, shard_base=shard_base)
        self.m = SpecModel(zmap, n, shard_base)
        for name in switches:
            getattr(self, "set_" + name)(True)
        self.dev = None
        self.timed_total = self.rtimed_total = self.started = self.listed = self.detailed = 0


def dry_queue(m, T, mode):
    """the candidate queue of the model's tick at T without committing it: (waiting slots in admission order, fresh
    slots ascending), local"""
    d = copy.copy(m)
    d.c = {k: v.copy() for k, v in m.c.items()}
    for name in ("since", "deadline", "rsince", "rdeadline", "wait", "wf", "spec_base"):
        setattr(d, name, getattr(m, name).copy())
    d.hc, d.rm = dict(m.hc), dict(m.rm)
    d.budget = ao.UNLIMITED
    out = d.tick(T, mode)
    loc = out.idx.astype(np.int64) - m.shard_base
    cand = loc[(out.act & np.uint32(ao.ACT_SUBMIT_HC)) != 0]
    waiting = m.wait[cand] != ao.NOT_WAITING
    w = cand[waiting]
    return w[np.lexsort((w, m.wait[w]))], np.sort(cand[~waiting])


def budget_for(cut, w, fresh, n, rng):
    """the budget that puts the cut where `cut` says, or None when this queue has no such place"""
    nw, groups, last = len(w), fresh // GROUP, (n - 1) // GROUP
    if cut == "zero":
        return 0
    if cut == "everyone":  # (no fresh candidate is deferred: adm_fresh_kernel's first uniform exit)
        return nw + len(fresh) + int(rng.integers(0, 3)) if len(np.unique(groups)) >= 2 else None
    if cut == "waiting":
        return int(rng.integers(1, nw)) if nw >= 2 else None
    if cut == "last_group":
        inside = int((groups == last).sum())
        return nw + int((groups < last).sum()) + int(rng.integers(1, inside)) if inside >= 2 else None
    # an edge with at least two fresh candidates on either side
    edges = [e for e in (int((groups < g).sum()) for g in range(1, last + 1)) if 2 <= e <= len(fresh) - 2]
    if not edges:
        return None
    return nw + edges[int(rng.integers(0, len(edges)))] + {"group_edge": 0, "before_edge": -1, "after_edge": 1}[cut]


def walk(am, zmap, entry, base, n=N, steps=STEPS, seed_text=""):
    rng = np.random.default_rng(zlib.crc32(f"admission scale {entry} {base} {seed_text}".encode()))
    T = M0 + 9 * DAY + 11 * 3600 - 2
    zones = zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))
    p = ScalePair(am, zmap, n, base, entry)

    def records(k):
        r = am.columns_to_records(population(rng, k, T, True, zones))
        r["wf_timeout"] = np.where(rng.random(k) < 0.5, 0, rng.integers(1, 300, k))
        return r

    reached = Counter()
    try:
        p.set_budget(1000)
        p.upsert(np.arange(n), records(n))
        for k, step in enumerate(steps):
            if k:
                waiting = np.flatnonzero(p.m.wait != ao.NOT_WAITING)
                busy = np.flatnonzero(p.m.since != NONE)
                ends = rng.choice(busy, min(len(busy), n // 6), replace=False)
                p.post(np.concatenate([ends, waiting[::7]]), rng.integers(0, 3, len(ends) + len(waiting[::7])),
                       rng.integers(0, 3, len(ends) + len(waiting[::7])).astype(np.uint8))
                sl = np.concatenate([rng.choice(n, 200, replace=False), waiting[1::11]])  # (an upsert keeps the wait)
                p.upsert(sl, records(len(sl)))
                sl = np.concatenate([rng.choice(n, 300, replace=False), waiting[2::13]])
                p.update_spec(sl, records(len(sl)))
                p.remove(np.concatenate([rng.choice(n, 40, replace=False), waiting[3::17]]))
                if k % 4 == 2:
                    p.load(int(rng.integers(0, n - 600)), population(rng, 600, T, True, zones))
            T += step
            mode = [0, CATCH, 0, FULL][k % 4]
            w, fresh = dry_queue(p.m, T, mode)
            # the least made cut this queue allows, in turn
            for cut in sorted(CUTS[k % len(CUTS):] + CUTS[:k % len(CUTS)], key=lambda c: reached[c]):
                b = budget_for(cut, w, fresh, n, rng)
                if b is not None:
                    reached[cut] += 1
                    break
            else:
                b = len(w) + len(fresh) // 2
            p.set_budget(b)
            p.tick(T, mode)
        return p, reached
    finally:
        p.close()


ENTRY_BASES = [(e, b) for b in (0, 12_345) for e in ("tick", "tick_short", "tick_view", "tick_device", "tick_shard")]


@pytest.mark.parametrize("entry,base", ENTRY_BASES + [("tick_device", (1 << 32) + 4_101)])
def test_budget_cuts_across_groups_equal_the_model(am, zmap, entry, base):
    p, reached = walk(am, zmap, entry, base)
    assert set(reached) == set(CUTS), reached
    assert p.detailed > 1000, p.detailed


def test_full_size_fifo_past_one_plan_round(am, zmap):
    """a backlog of more FIFO entries than one round of the plan's scan covers (1024 chunks of 256): 300,000 interval
    checks due at once under a budget of 1000, then ticks whose posts and removes end waits scattered through the FIFO
    under budgets that keep it over 262,144 entries; every tick against the model"""
    if emulated(am):
        pytest.skip("300,000 records: the GPU")
    n = 300_000
    rng = np.random.default_rng(11)
    T = M0 + 3 * DAY + 5
    p = ScalePair(am, zmap, n, 7, "tick")
    try:
        p.set_budget(1000)
        r = am.columns_to_records(population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY))))
        due = rec(am, 0, repeat_after_sec=30, finished_at=T - 1000)
        r[rng.random(n) < 0.95] = due  # (nearly all due at the first tick)
        p.upsert(np.arange(n), r)
        sizes = []
        for k, step in enumerate([0, 1, 1, 59, 1, 60]):
            if k:
                waiting = np.flatnonzero(p.m.wait != ao.NOT_WAITING)
                busy = np.flatnonzero(p.m.since != NONE)
                p.post(np.concatenate([busy[::3], waiting[::97]]), np.full(len(busy[::3]) + len(waiting[::97]), 1))
                p.remove(waiting[5::89])
                p.set_budget([3000, 0, 5000, 2000, 1000][k - 1])
            T += step
            p.tick(T)
            sizes.append(p.s.last_admission()["n_deferred"])
        assert sum(s > 262_144 for s in sizes) >= 4, sizes
    finally:
        p.close()


def _backlog_pair(am, zmap, rng, T, n=N, base=0, switches=("hold", "remedy")):
    """a pair at the scale shape with a backlog of waits spread over every group"""
    p = ScalePair(am, zmap, n, base, "tick", switches)
    zones = zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))
    r = am.columns_to_records(population(rng, n, T, True, zones))
    r["wf_timeout"] = np.where(rng.random(n) < 0.5, 0, rng.integers(1, 300, n))
    p.upsert(np.arange(n), r)
    p.set_budget(300)
    for k, step in enumerate([0, 1, 60, 1]):
        T += step
        if k == 2:
            busy = np.flatnonzero(p.m.since != NONE)
            p.post(busy[::2], rng.integers(1, 3, len(busy[::2])))
        p.tick(T)
    waiting = np.flatnonzero(p.m.wait != ao.NOT_WAITING)
    assert len(np.unique(waiting // GROUP)) == (n - 1) // GROUP + 1, "a wait in every group"
    return p, T


def _shard_model(zmap, m, lo, hi):
    """the model of slots [lo, hi) of `m` as a handle at shard_base lo that restored them holds them"""
    t = SpecModel(zmap, hi - lo, lo, hold=True, remedy=m.remedy)
    for name, col in t.c.items():
        col[:] = m.c[name][lo:hi]
    for name in ("since", "deadline", "rsince", "rdeadline", "wait", "wf"):
        getattr(t, name)[:] = getattr(m, name)[lo:hi]
    t.hwm, t.P, t.adm = hi - lo, m.P, True
    return t


def test_checkpoint_mid_backlog_into_three_shards_keeps_finite_budgets(am, zmap):
    """a checkpoint taken mid-backlog, cut at bounds off group and word edges, restored into three handles: each keeps a
    finite budget of its own and goes on tick for tick as the source's model cut to its slots does"""
    rng = np.random.default_rng(41)
    p, T = _backlog_pair(am, zmap, rng, M0 + 2 * DAY + 7 * 3600 - 3)
    bounds = [0, GROUP + 1013, 2 * GROUP + 4099, N]  # (neither a multiple of 8192 nor of 32)
    assert all(b % 32 for b in bounds[1:-1])
    shards = []
    try:
        for k, (lo, hi) in enumerate(zip(bounds, bounds[1:])):
            blob = p.s.checkpoint(lo, hi - lo)
            q = ScalePair(am, zmap, hi - lo, lo, "tick", ("hold", "remedy"))
            q.set_budget(0)
            q.s.restore(blob)
            q.m = _shard_model(zmap, p.m, lo, hi)
            np.testing.assert_array_equal(q.s.deferred(0, hi - lo), q.m.deferred(0, hi - lo))
            q.set_budget([5, 40, 0][k])
            shards.append(q)
        for j, step in enumerate([1, 59, 1, 1, 60]):
            T += step
            for k, q in enumerate(shards):
                busy = np.flatnonzero(q.m.since != NONE)
                q.post(busy[::3], rng.integers(1, 3, len(busy[::3])))
                if j == 2:
                    q.set_budget([100, 7, 30][k])
                q.tick(T)
        assert all(q.m.last_admission()["n_deferred"] > 0 for q in shards)
    finally:
        for q in shards:
            q.close()
        p.close()


def test_simulate_tick_by_tick_under_a_budget_at_scale(am, zmap):
    """am_sweep_simulate under finite budgets on the scale shape: tests/sim_driver.py's loop of posts and ticks on the
    model, per-tick statistics and simulation rows, then the columns, the runs in flight, the waits and the last
    admission"""
    rng = np.random.default_rng(43)
    p, T = _backlog_pair(am, zmap, rng, M0 + 4 * DAY + 3600 - 5)
    params, seed = (2, 9, 3, 12), 79
    try:
        for budget in (300, 0, 2000):
            p.set_budget(budget)
            T += 1
            wrows, wsims = sim_driver.simulate(p.m, T, 12, 0, seed, params)
            rows, sims = p.s.simulate(T, 12, 0, seed, params)
            for k, (r, w) in enumerate(zip(rows, wrows)):
                gd = {f: int(r[f]) for f in am.abi.STAT_FIELDS}
                assert gd == w, (budget, k, {f: (gd[f], w[f]) for f in gd if gd[f] != w[f]})
            np.testing.assert_array_equal(np.array([tuple(x) for x in sims], dtype=np.int64).reshape(-1, 4),
                                          np.array(wsims, dtype=np.int64).reshape(-1, 4))
            p.m.drained()
            dev = p.s.read_range(0, N)
            for name in am.COLUMN_NAMES:
                np.testing.assert_array_equal(dev[name], p.m.cols()[name], err_msg=f"{budget}: {name}")
            np.testing.assert_array_equal(p.s.in_flight(0, N), p.m.in_flight(0, N))
            np.testing.assert_array_equal(p.s.deferred(0, N), p.m.deferred(0, N))
            assert p.s.last_admission() == p.m.last_admission()
            T += 12
    finally:
        p.close()


def test_full_size_1026_groups(am, zmap):
    """1025 * 8192 + 1000 records (1026 groups, more than one round of the plan's group scan): three ticks against the
    model, each with its budget from the dry run, one of them cutting inside a group >= 1024"""
    if emulated(am):
        pytest.skip("8.4 M records: the GPU")
    n = 1025 * GROUP + 1000
    rng = np.random.default_rng(47)
    T = M0 + 6 * DAY + 5
    p = ScalePair(am, zmap, n, 0, "tick", ("hold",))
    try:
        r = am.columns_to_records(population(rng, n, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY))))
        r[rng.random(n) < 0.3] = rec(am, 0, repeat_after_sec=30, finished_at=T - 1000)
        p.upsert(np.arange(n), r)
        p.set_budget(50_000)
        cut_groups = []
        for k, step in enumerate([0, 1, 60]):
            T += step
            if k:
                busy = np.flatnonzero(p.m.since != NONE)
                p.post(busy[::2], np.full(len(busy[::2]), 1))
            w, fresh = dry_queue(p.m, T, 0)
            late = int((fresh < 1024 * GROUP).sum())
            assert late < len(fresh), "fresh candidates in the last groups"
            b = len(w) + late + int(rng.integers(0, len(fresh) - late))  # (a cut inside group >= 1024)
            cut_groups.append(int(fresh[b - len(w)] // GROUP))
            p.set_budget(b)
            p.tick(T)
        assert (n - 1) // GROUP + 1 == 1026 and min(cut_groups) >= 1024, cut_groups
    finally:
        p.close()


def test_one_gpu_world_exchange_of_a_budgeted_shard(am, zmap):
    """the admitted list through the exchange of a one-GPU world: a budgeted handle at a base past 2^32 bound to
    gather.PeerGather with u64 indices; after each whole step (tick_view) the global list and the view equal the
    model's list, the statistics, waits and last admission the model's"""
    import importlib
    gather = importlib.import_module("active-monitor_b200.gather")
    base = (1 << 32) + 777
    rng = np.random.default_rng(53)
    T = M0 + 7 * DAY + 11 * 3600 - 1
    p = ScalePair(am, zmap, N, base, "tick", ("hold", "remedy"))
    g = gather.PeerGather(0, cap_total=N, idx_bytes=8, shard=(base, N))
    try:
        p.upsert(np.arange(N), am.columns_to_records(population(rng, N, T, True,
                                                                 zmap.ids_of(zones_usable(T - DAY, T + DAY)))))
        g.bind(p.s)
        for k, step in enumerate([0, 1, 59, 1, 60, 1]):
            T += step
            p.set_budget([200, 0, 35, 1000, 7, None][k])
            if k:
                busy = np.flatnonzero(p.m.since != NONE)
                p.post(busy[::2], rng.integers(1, 3, len(busy[::2])))
                sl = rng.choice(N, 100, replace=False)
                p.update_spec(sl, am.columns_to_records(population(rng, 100, T, True, zmap.ids_of(zones_usable(T - DAY, T + DAY)))))
            want = p.m.tick(T, 0)
            vi, va, st = g.tick_view(T, 0)
            np.testing.assert_array_equal(vi.astype(np.uint64) + np.uint64(base), want.idx, err_msg=f"{k}: view")
            np.testing.assert_array_equal(va.astype(np.uint32), want.act, err_msg=f"{k}: view act")
            gi, ga, counts = g.result()
            assert counts == [len(want.idx)], (k, counts)
            np.testing.assert_array_equal(gi.cpu().numpy().astype(np.uint64), want.idx, err_msg=f"{k}: global idx")
            np.testing.assert_array_equal(ga.cpu().numpy().astype(np.uint32), want.act, err_msg=f"{k}: global act")
            assert {f: int(st[f]) for f in want.stats} == want.stats, k
            np.testing.assert_array_equal(p.s.deferred(0, N), p.m.deferred(0, N), err_msg=f"{k}: deferred")
            if p.m.adm:
                assert p.s.last_admission() == p.m.last_admission(), k
        assert p.m.admission["n_deferred"] >= 0
    finally:
        g.close()
        p.close()
