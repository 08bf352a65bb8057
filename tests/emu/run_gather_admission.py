"""Child process of tests/test_admission_exchange_emulator.py: the submit budget through the sharded whole step on the
rank harness (tests/emu/ranks.py).  Every rank has the hold on, its own budget and its own model
(tests/spec_update_model.py at the rank's shard_base).  Between steps posts and spec updates are sent to the rank that
owns the slot, and the ranks' budgets change.  After every am_gather_tick_view each rank's global list must equal the
concatenation, in rank order, of the ranks' models' lists; its view its own part; its statistics its model's; and its
waits (deferred) and last admission its model's.

usage: run_gather_admission.py <world> <idx_bytes> <records in total> <config>
Prints "ok ..." and exits 0 on success."""
import sys

import numpy as np
from ranks import HOLD_TICKS, Gather, Shards, abi, am, check_list, check_view, population, run_ranks

import admission_oracle as ao  # noqa: E402
from handle_model import NONE  # noqa: E402
from spec_update_model import SpecModel  # noqa: E402

world, idx_bytes, n_total, config = (int(a) for a in sys.argv[1:5])
zmap, whole = population(n_total, config)
lay = Shards(n_total, world)
BUDGETS = [0, 3, 17, 60, 400, None]

# the models run first: they decide the posts before each step; every rank replays its own calls
rng = np.random.default_rng(world * 1000 + config)
models = []
for r in range(world):
    m = SpecModel(zmap, int(lay.sizes[r]), int(lay.bases[r]), hold=True)
    m.load(0, lay.part(whole, r))
    models.append(m)
calls = [[[] for _ in HOLD_TICKS] for _ in range(world)]  # per rank, per step: (name, args)
want = []  # per step: (global idx, act) and per rank (stats, deferred, last admission)
for k, (T, mode) in enumerate(HOLD_TICKS):
    for r, m in enumerate(models):
        if k % 3 == 0:
            calls[r][k].append(("set_budget", (BUDGETS[int(rng.integers(0, len(BUDGETS)))] if k else 20,)))
        if k:
            busy = np.flatnonzero(m.since != NONE)
            sl = rng.choice(busy, min(len(busy), 40), replace=False)
            calls[r][k].append(("post", (sl, rng.integers(1, 3, len(sl)).astype(np.uint8))))
            src = rng.integers(0, n_total, 30)
            recs = am.columns_to_records({c: v[src] for c, v in whole.items()})
            calls[r][k].append(("update_spec", (rng.choice(m.capacity, 30, replace=False), recs)))
        for name, args in calls[r][k]:
            getattr(m, name)(*args)
    outs = [m.tick(T, mode) for m in models]
    want.append((np.concatenate([o.idx for o in outs]), np.concatenate([o.act for o in outs]),
                 [(o.stats, m.deferred(), m.last_admission()) for o, m in zip(outs, models)]))
deferred = sum(w[2][r][2]["n_deferred"] for w in want for r in range(world))
assert deferred > 0, deferred


def rank_main(rank, bar):
    first, cnt = lay.shards[rank]
    s = am.Sweep(capacity=cnt, device=rank, shard_base=first)
    s.set_hold_in_flight(True)
    s.load_range(0, lay.part(whole, rank))
    g = Gather.bound(rank, bar, lay, s, idx_bytes)
    for k, (T, mode) in enumerate(HOLD_TICKS):
        for name, args in calls[rank][k]:
            if name == "set_budget":
                s.set_submit_budget(args[0])
            elif name == "post":
                s.post_result(*args)
            else:
                s.update_spec(*args)
        gi, ga, _, vw = g.step(T, mode)
        wi, wa, per_rank = want[k]
        check_list(rank, k, gi, ga, wi, wa)
        part = lay.own(wi, rank)
        check_view(rank, k, vw, wi[part], wa[part])
        stats, dfr, adm = per_rank[rank]
        got = {f: int(g.st[f][0]) for f in abi.STAT_FIELDS}
        assert got == stats, (rank, k, {f: (got[f], stats[f]) for f in got if got[f] != stats[f]})
        np.testing.assert_array_equal(s.deferred(0, cnt), dfr, err_msg=f"rank {rank} step {k} deferred")
        assert s.last_admission() == adm, (rank, k, s.last_admission(), adm)
    g.close(bar, s)


run_ranks(world, rank_main)
print(f"ok admission world={world} idx_bytes={idx_bytes} n={n_total} config={config} deferred={deferred} "
      f"emitted={[len(w[0]) for w in want]} waiting={[int((m.wait != ao.NOT_WAITING).sum()) for m in models]}")
