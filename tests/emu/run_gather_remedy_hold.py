"""Child process of tests/test_remedy_hold_emulator.py: the remedy hold through the sharded whole step, as
run_gather_timeout.py runs workflow timeouts, with half of the records on a remedy workflow and the remedy hold on
(the remedy variants of am_sweep_tick_shard).  Between ticks a few workflow phases are posted for checks in flight and
a few remedy phases for running remedies, each to the rank that owns it; the rest time out.  Every rank's global list
must equal the remedy-hold oracle (tests/remedy_hold_oracle.py) of the UNSHARDED population, its view, its
am_sweep_last_timed_out and its am_sweep_last_remedy_timed_out the part it owns; at the end its columns,
am_sweep_in_flight and am_sweep_remedy_in_flight the oracle's.

usage: run_gather_remedy_hold.py <world> <idx_bytes> <records in total> <config>
Prints "ok ..." and exits 0 on success."""
import sys

import numpy as np
from ranks import HOLD_TICKS, Gather, Shards, abi, am, check_columns, check_list, check_view, lib, population, run_ranks

from handle_model import NONE, HandleModel  # noqa: E402

world, idx_bytes, n_total, config = (int(a) for a in sys.argv[1:5])
zmap, whole = population(n_total, config, remedy=True)
lay = Shards(n_total, world)

# the model run first: it decides which in-flight checks post a phase before each tick
rng = np.random.default_rng(world * 1000 + config)
wf = np.random.default_rng(world * 77 + config).integers(0, 120, n_total).astype(np.int32)
model = HandleModel(zmap, n_total, hold=True, remedy=True)
recs = am.columns_to_records(whole)
recs["wf_timeout"] = wf
model.upsert(np.arange(n_total), recs)
want, posts = [], []
for k, (T, mode) in enumerate(HOLD_TICKS):
    fl = np.flatnonzero(model.since != NONE)
    sl = np.sort(rng.choice(fl, min(len(fl), 60), replace=False)) if k and len(fl) else np.zeros(0, np.int64)
    ph = rng.integers(1, 3, len(sl)).astype(np.uint8)  # replaced below, but its draw fixes the later ones
    ph = np.where(rng.random(len(sl)) < 0.8, 2, 1).astype(np.uint8)
    model.post(sl, ph)
    rl = np.flatnonzero(model.rsince != NONE)
    rl = np.sort(rng.choice(rl, min(len(rl), 20), replace=False)) if len(rl) else np.zeros(0, np.int64)
    model.post(rl, np.zeros(len(rl), np.uint8), np.ones(len(rl), np.uint8))
    posts.append((sl, ph, rl))
    want.append(model.tick(T, mode))
assert sum(int(((w[1] & abi.ACT_SUBMIT_HC) != 0).sum()) for w in want[1:]) > 0
assert sum(len(w[3][0]) for w in want) > 100 and sum(len(w[4][0]) for w in want) > 20
n_timed = [0] * world
n_rtimed = [0] * world


def rank_main(rank, bar):
    first, cnt = lay.shards[rank]
    s = am.Sweep(capacity=cnt, device=rank, shard_base=first)
    s.set_hold_in_flight(True)
    s.set_hold_remedy(True)
    recs = am.columns_to_records(lay.part(whole, rank))
    recs["wf_timeout"] = wf[first:first + cnt]
    s.upsert(np.arange(cnt), recs)
    g = Gather.bound(rank, bar, lay, s, idx_bytes)
    for k, (T, mode) in enumerate(HOLD_TICKS):
        sl, ph, rl = posts[k]
        own = lay.own(sl, rank)
        if own.any():
            s.post_result(sl[own] - first, ph[own])
        own = lay.own(rl, rank)
        if own.any():
            s.post_result(rl[own] - first, np.zeros(int(own.sum()), np.uint8), np.ones(int(own.sum()), np.uint8))
        gi, ga, _, vw = g.step(T, mode)
        wi, wa, _, timed, rtimed = want[k]
        check_list(rank, k, gi, ga, wi, wa)
        part = lay.own(wi, rank)
        check_view(rank, k, vw, wi[part], wa[part])
        ti, ts = s.last_timed_out()
        mine = lay.own(timed[0], rank)
        np.testing.assert_array_equal(ti, timed[0][mine], err_msg=f"rank {rank} tick {k} timed out")
        np.testing.assert_array_equal(ts, timed[1][mine], err_msg=f"rank {rank} tick {k} timed-out since")
        n_timed[rank] += len(ti)
        ri, rs = s.last_remedy_timed_out()
        mine = lay.own(rtimed[0], rank)
        np.testing.assert_array_equal(ri, rtimed[0][mine], err_msg=f"rank {rank} tick {k} remedy timed out")
        np.testing.assert_array_equal(rs, rtimed[1][mine], err_msg=f"rank {rank} tick {k} remedy start")
        n_rtimed[rank] += len(ri)
    bar.wait()
    check_columns(rank, s, lay.part(model.cols(), rank))
    np.testing.assert_array_equal(s.in_flight(0, cnt), model.in_flight()[first:first + cnt],
                                  err_msg=f"rank {rank} in_flight")
    np.testing.assert_array_equal(s.remedy_in_flight(0, cnt), model.remedy_in_flight()[first:first + cnt],
                                  err_msg=f"rank {rank} remedy_in_flight")
    # a closed-loop step is refused on every rank before anything happens (no exchange needed)
    rc = lib.am_sweep_tick_shard(s._h, HOLD_TICKS[-1][0] + 1, abi.SWEEP_CLOSED_LOOP, None)
    assert rc == abi.AM_E_INVAL, (rank, rc)
    g.close(bar, s)


run_ranks(world, rank_main)
assert all(v > 0 for v in n_rtimed), n_rtimed  # every shard timed out remedy runs of its own
print(f"ok remedy hold remedy_timed_out_per_rank={n_rtimed} timed_out_per_rank={n_timed} world={world} idx_bytes={idx_bytes} n={n_total} config={config} "
      f"emitted={[len(w[0]) for w in want]} remedy_held={int((model.remedy_in_flight() != NONE).sum())}")
