"""Child process of the emulator tests: `world` ranks drive the exchange through the rank harness (tests/emu/ranks.py).

usage: run_gather_ranks.py tick  <world> <idx_bytes> <records in total> <ticks> [config]
       run_gather_ranks.py plain <world> <idx_bytes> <records per rank> <ticks>

tick : every rank owns an index-range shard of ONE amgen population (am.Sweep on its own "device"),
       per tick am_sweep_tick_shard + am_gather_exchange, no barrier between ticks; every rank's
       global list, counts and shard statistics must equal the UNSHARDED oracle sweep, and the
       shard's columns the oracle's columns at the end.
       EMU_ABSENT_RANK=r: rank r never exchanges; the others must report the watchdog value.
       EMU_TICK_VIEW=1: the step through am_gather_bind + am_gather_tick_view; the view must be the rank's own
       part of the list as local slots.
plain: the round-1 list format (am_gather_push) against the concatenation of random lists.
Prints "ok ..." and exits 0 on success."""
import ctypes as C
import os
import sys

import numpy as np
from ranks import Gather, Shards, abi, am, check_columns, check_list, check_view, lib, run_ranks

import amgen  # noqa: E402
import oracle_c  # noqa: E402

mode, world, idx_bytes, n_arg, ticks = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5])
config = int(sys.argv[6]) if len(sys.argv) > 6 else 3
T0 = 1789982100
absent = int(os.environ.get("EMU_ABSENT_RANK", "-1"))
use_view = os.environ.get("EMU_TICK_VIEW") == "1"  # am_gather_tick_view instead of tick_shard + exchange


# ---------------------------------------------------------------- tick exchange
if mode == "tick":
    n_total = n_arg
    lay = Shards(n_total, world)
    whole = amgen.fill(config, 4, 0, n_total, T0, oracle_c.load().orc_classify, threads=2)
    want = []  # per tick: (T, idx, act)
    for k in range(ticks):
        T = T0 + 60 * k - (k % 2)  # on and off the minute
        wi, wa, _ = oracle_c.sweep(whole, T)
        want.append((T, wi, wa))

    def rank_main(rank, bar):
        first, cnt = lay.shards[rank]
        cols = amgen.fill(config, 4, first, cnt, T0, lib.am_healthcheck_classify, threads=1)
        ocols = {k: v.copy() for k, v in cols.items()}
        s = am.Sweep(capacity=cnt, device=rank, shard_base=first)
        s.load_range(0, cols)
        g = Gather(rank, bar, n_total, idx_bytes)
        g.set_layout(lay)
        # argument errors come back before anything a peer could observe happens
        assert lib.am_gather_exchange(g.h, s._h, None, None) == abi.AM_E_INVAL  # no tick_shard yet
        if use_view:
            assert lib.am_gather_tick_view(g.h, T0, 0, C.byref(abi.AmTickView()), None) == abi.AM_E_INVAL  # not bound yet
            g.bind(s)

        def exchange(T):
            s.tick_shard(T)
            rc = lib.am_gather_exchange(g.h, s._h, g.st.ctypes.data, None)
            assert rc == 0, (rc, lib.am_gather_last_error(g.h))

        for k, (T, wi, wa) in enumerate(want if rank != absent else []):  # no barrier between ticks, as on a stream
            if absent >= 0:  # a peer never arrives: the watchdog value, which the whole step reports as an error
                if use_view:
                    rc = g.tick_view(T, 0)[0]
                    assert rc == abi.AM_E_DEVICE, rc
                else:
                    exchange(T)
                counts = g.counts()
                assert int(counts[world]) == 0xFFFFFFFF, counts
                break
            if use_view:  # the whole step in one call (am_gather_bind + am_gather_tick_view)
                gi, ga, counts, vw = g.step(T, 0)
            else:
                exchange(T)
                gi, ga, counts = g.read()
            check_list(rank, k, gi, ga, wi, wa)
            oi, oa, ost = oracle_c.sweep(ocols, T, shard_base=first)  # this shard alone
            got = {f: int(g.st[f][0]) for f in abi.STAT_FIELDS}
            assert got == ost, (rank, k, got, ost)
            if use_view:  # this rank's own part of the global list
                check_view(rank, k, vw, oi, oa)
            assert [int(c) for c in counts[:world]] == [int(lay.own(wi, r).sum()) for r in range(world)]
        if absent < 0:
            check_columns(rank, s, ocols)
        g.close(bar, s)

# ---------------------------------------------------------------- plain lists
else:
    n_rec = n_arg
    sizes_l = [n_rec + (37 if r == world - 1 else 0) for r in range(world)]
    bases = np.concatenate([[0], np.cumsum(sizes_l)[:-1]]).astype(np.uint64)

    def local_list(rank, tick):
        rng = np.random.default_rng(1000 * tick + rank)
        emitted = rng.random(sizes_l[rank]) < (0.33 if (tick + rank) % 3 else 0.9)
        if tick % 4 == 3 and rank == 1:
            emitted[:] = False
        idx = np.flatnonzero(emitted).astype(np.uint32)
        act = np.where(rng.random(len(idx)) < 0.97, 0x01, rng.choice([0x08, 0x23, 0x80], len(idx))).astype(np.uint8)
        return idx, act

    def rank_main(rank, bar):
        g = Gather(rank, bar, int(sum(sizes_l)), idx_bytes)
        for t in range(1, ticks + 1):
            idx, act = local_list(rank, t)
            cnt = np.array([len(idx)], dtype=np.uint32)
            idx_buf = np.concatenate([idx, np.zeros(4, np.uint32)])  # device buffers are larger than the list
            act_buf = np.concatenate([act, np.zeros(4, np.uint8)])
            rc = lib.am_gather_push(g.h, idx_buf.ctypes.data, act_buf.ctypes.data, cnt.ctypes.data, int(bases[rank]), None)
            assert rc == 0, (rc, lib.am_gather_last_error(g.h))
            gi, ga, counts = g.read()
            want_i, want_a = [], []
            for r in range(world):
                li, la = local_list(r, t)
                assert int(counts[r]) == len(li), (rank, t, r, int(counts[r]), len(li))
                want_i.append(li.astype(np.uint64) + bases[r])
                want_a.append(la)
            check_list(rank, t, gi, ga, np.concatenate(want_i), np.concatenate(want_a))
        g.close(bar)


run_ranks(world, rank_main)
print(f"ok {mode}{' watchdog' if absent >= 0 else ''} world={world} idx_bytes={idx_bytes} n={n_arg} ticks={ticks}")
