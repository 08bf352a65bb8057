"""Child process of tests/test_catch_up_exchange_emulator.py: catch-up ticks (AM_SWEEP_CATCH_UP) through the sharded
whole step, on the rank harness (tests/emu/ranks.py): every rank owns an index-range shard of ONE amgen population and
calls am_gather_tick_view (am_sweep_tick_shard, the window variant launched without programmatic dependent launch, then
the exchange of its bitmap, exceptions and statistics).  A plain tick sets P, then catch-up ticks follow whose windows
hold no minute start, cross a minute, cross an hour and span a whole day across midnight.  Every rank's global list
must equal the window oracle of the UNSHARDED population (tests/window_oracle.py), its view and shard statistics the
window oracle of its shard alone, its columns the oracle's at the end; afterwards every rank's P must be the last tick's
second.

usage: run_gather_catch_up.py <world> <idx_bytes> <records in total> <config> <closed 0|1>
Prints "ok ..." and exits 0 on success."""
import sys

from ranks import T0, Gather, Shards, abi, am, check_columns, check_list, check_view, lib, population, run_ranks

import window_oracle  # noqa: E402

world, idx_bytes, n_total, config, closed = (int(a) for a in sys.argv[1:6])
mode = abi.SWEEP_CLOSED_LOOP if closed else 0
SEED = 5
TICKS = [(T0, False),                    # plain: sets P
         (T0 + 9, True),                 # (23:44:50, 23:44:59]: no minute start, the plain sweep
         (T0 + 9 + 61, True),            # crosses 23:45:00 and 23:46:00
         (T0 + 70 + 3607, True),         # an hour, across midnight
         (T0 + 3677 + 86400, True)]      # a whole day

zmap, whole = population(n_total, config)
lay = Shards(n_total, world)


def oracle_run(cols, shard_base):
    """per tick (idx, act, stats) of the oracle over `cols` (in place)"""
    out, P = [], None
    for T, catch_up in TICKS:
        if catch_up:
            out.append(window_oracle.sweep_window(zmap, cols, P, T, mode=mode, seed=SEED, shard_base=shard_base))
        else:
            out.append(zmap.sweep(cols, T, mode=mode, seed=SEED, shard_base=shard_base))
        P = T
    return out


want = oracle_run({k: v.copy() for k, v in whole.items()}, 0)
shard_cols = [lay.part(whole, r) for r in range(world)]
shard_want = [oracle_run(shard_cols[r], lay.shards[r][0]) for r in range(world)]


def rank_main(rank, bar):
    first, cnt = lay.shards[rank]
    s = am.Sweep(capacity=cnt, device=rank, shard_base=first)
    s.load_range(0, lay.part(whole, rank))
    s.set_seed(SEED)
    g = Gather.bound(rank, bar, lay, s, idx_bytes)
    for k, (T, catch_up) in enumerate(TICKS):
        gi, ga, _, vw = g.step(T, mode | (abi.SWEEP_CATCH_UP if catch_up else 0))
        check_list(rank, k, gi, ga, *want[k][:2])
        oi, oa, ost = shard_want[rank][k]
        got = {f: int(g.st[f][0]) for f in abi.STAT_FIELDS}
        assert got == ost, (rank, k, got, ost)
        check_view(rank, k, vw, oi, oa)
    bar.wait()
    check_columns(rank, s, shard_cols[rank])
    # P is the last tick's second on every rank: a day and a second later is refused, without effect (no exchange
    # needed), a day later is accepted
    last = TICKS[-1][0]
    rc = lib.am_sweep_tick_shard(s._h, last + 86401, mode | abi.SWEEP_CATCH_UP, None)
    assert rc == abi.AM_E_RANGE, (rank, rc)
    rc = lib.am_sweep_tick_shard(s._h, last + 86400, mode | abi.SWEEP_CATCH_UP, None)
    assert rc == 0, (rank, rc)
    g.close(bar, s)


run_ranks(world, rank_main)
print(f"ok catch-up world={world} idx_bytes={idx_bytes} n={n_total} config={config} closed={closed} "
      f"emitted={[len(w[0]) for w in want]}")
