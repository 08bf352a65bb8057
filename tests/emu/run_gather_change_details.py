"""Child process of tests/test_change_details_emulator.py: change details through the sharded whole step, as
run_gather_changes.py runs the status changes, with tracking and details on.  Between ticks results are posted,
each to the rank that owns its slot (one tick's batch dense enough for the sweep to apply it), and some ranks read in
between.  Every rank's global list must equal the oracle of the UNSHARDED population, and its
am_sweep_last_change_details the part of the change-details oracle (tests/change_details_oracle.py) it owns.

usage: run_gather_change_details.py <world> <idx_bytes> <records in total> <config>
Prints "ok ..." and exits 0 on success."""
import sys

import numpy as np
from ranks import CHANGE_TICKS, Gather, Shards, am, check_list, population, run_ranks

import change_details_oracle  # noqa: E402
from handle_model import HandleModel  # noqa: E402

world, idx_bytes, n_total, config = (int(a) for a in sys.argv[1:5])
zmap, whole = population(n_total, config, remedy=True)
lay = Shards(n_total, world)

rng = np.random.default_rng(world * 1000 + config)
model = HandleModel(zmap, n_total, track=True, details=True)
model.upsert(np.arange(n_total), am.columns_to_records(whole))
want, posts = [], []
for k, (T, mode) in enumerate(CHANGE_TICKS):
    m = n_total // 4 if k == 3 else 200  # tick 3: more than an eighth of the records, applied inside the sweep
    sl = np.sort(rng.choice(n_total, m, replace=False)) if k else np.zeros(0, np.int64)
    ph = rng.integers(0, 3, len(sl)).astype(np.uint8)
    rp = rng.integers(0, 3, len(sl)).astype(np.uint8)
    model.post(sl, ph, rp)
    posts.append((sl, ph, rp))
    out = model.tick(T, mode)
    want.append((out[0], out[1], model.changes(), model.details().copy()))
assert sum(len(w[2]) for w in want) > n_total // 8
listed = [0] * world


def rank_main(rank, bar):
    first, cnt = lay.shards[rank]
    s = am.Sweep(capacity=cnt, device=rank, shard_base=first)
    s.set_track_changes(True)
    s.set_change_details(True)
    s.upsert(np.arange(cnt), am.columns_to_records(lay.part(whole, rank)))
    g = Gather.bound(rank, bar, lay, s, idx_bytes)
    for k, (T, mode) in enumerate(CHANGE_TICKS):
        sl, ph, rp = posts[k]
        own = lay.own(sl, rank)
        if own.any():
            s.post_result(sl[own] - first, ph[own], rp[own])
            if (rank + k) % 2:  # a read leaves them pending for the tick
                s.read(sl[own][:5] - first)
        gi, ga = g.step(T, mode)[:2]
        wi, wa, wc, wdet = want[k]
        check_list(rank, k, gi, ga, wi, wa)
        ci, cd = s.last_change_details()
        part = lay.own(wc, rank)
        np.testing.assert_array_equal(ci, wc[part], err_msg=f"rank {rank} tick {k} changes")
        for name in change_details_oracle.DETAIL.names:
            np.testing.assert_array_equal(cd[name], wdet[name][part], err_msg=f"rank {rank} tick {k} {name}")
        listed[rank] += len(ci)
    g.close(bar, s)


run_ranks(world, rank_main)
assert all(v > 0 for v in listed), listed
print(f"ok change details listed_per_rank={listed} world={world} idx_bytes={idx_bytes} n={n_total} config={config} "
      f"changed={[len(w[2]) for w in want]}")
