"""Child process of tests/test_in_flight_exchange_emulator.py: ticks with the hold in flight on, through the sharded
whole step on the rank harness (tests/emu/ranks.py): the hold variants of am_sweep_tick_shard, then the exchange.
Between ticks Succeeded / Failed phases are posted for some of the checks in flight, each to the rank that owns it.  Every rank's global list must equal the hold oracle
(tests/hold_oracle.py) of the UNSHARDED population, its view the part of that list it owns; at the end its columns and
am_sweep_in_flight the oracle's.

usage: run_gather_hold.py <world> <idx_bytes> <records in total> <config>
Prints "ok ..." and exits 0 on success."""
import sys

import numpy as np
from ranks import HOLD_TICKS, Gather, Shards, abi, am, check_columns, check_list, check_view, lib, population, run_ranks

from handle_model import NONE, HandleModel  # noqa: E402

world, idx_bytes, n_total, config = (int(a) for a in sys.argv[1:5])
zmap, whole = population(n_total, config)
lay = Shards(n_total, world)

# the model run first: it decides which in-flight checks post a phase before each tick
rng = np.random.default_rng(world * 1000 + config)
model = HandleModel(zmap, n_total, hold=True)
model.load(0, whole)
want, posts = [], []
for k, (T, mode) in enumerate(HOLD_TICKS):
    fl = np.flatnonzero(model.since != NONE)
    sl = np.sort(rng.choice(fl, min(len(fl), 300), replace=False)) if k and len(fl) else np.zeros(0, np.int64)
    ph = rng.integers(1, 3, len(sl)).astype(np.uint8)
    model.post(sl, ph)
    posts.append((sl, ph))
    want.append(model.tick(T, mode))
assert sum(int(((w[1] & abi.ACT_SUBMIT_HC) != 0).sum()) for w in want[1:]) > 0


def rank_main(rank, bar):
    first, cnt = lay.shards[rank]
    s = am.Sweep(capacity=cnt, device=rank, shard_base=first)
    s.set_hold_in_flight(True)
    s.load_range(0, lay.part(whole, rank))
    g = Gather.bound(rank, bar, lay, s, idx_bytes)
    for k, (T, mode) in enumerate(HOLD_TICKS):
        sl, ph = posts[k]
        own = lay.own(sl, rank)
        if own.any():
            s.post_result(sl[own] - first, ph[own])
        gi, ga, _, vw = g.step(T, mode)
        wi, wa = want[k][:2]
        check_list(rank, k, gi, ga, wi, wa)
        part = lay.own(wi, rank)
        check_view(rank, k, vw, wi[part], wa[part])
    bar.wait()
    check_columns(rank, s, lay.part(model.cols(), rank))
    np.testing.assert_array_equal(s.in_flight(0, cnt), model.in_flight()[first:first + cnt],
                                  err_msg=f"rank {rank} in_flight")
    # a closed-loop step is refused on every rank before anything happens (no exchange needed)
    rc = lib.am_sweep_tick_shard(s._h, HOLD_TICKS[-1][0] + 1, abi.SWEEP_CLOSED_LOOP, None)
    assert rc == abi.AM_E_INVAL, (rank, rc)
    g.close(bar, s)


run_ranks(world, rank_main)
print(f"ok hold world={world} idx_bytes={idx_bytes} n={n_total} config={config} "
      f"emitted={[len(w[0]) for w in want]} held={int((model.since != NONE).sum())}")
