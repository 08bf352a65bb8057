"""Child process of tests/test_catch_up_exchange_emulator.py: catch-up ticks (AM_SWEEP_CATCH_UP) through the sharded
whole step.  `world` ranks as Python threads drive the REAL C-ABI of the emulated library, as run_gather_ranks.py
does: every rank owns an index-range shard of ONE amgen population and calls am_gather_tick_view (am_sweep_tick_shard,
the window variant launched without programmatic dependent launch, then the exchange of its bitmap, exceptions and
statistics).  A plain tick sets P, then catch-up ticks follow whose windows hold no minute start, cross a minute,
cross an hour and span a whole day across midnight.  Every rank's global list must equal the window oracle of the
UNSHARDED population (tests/window_oracle.py), its view and shard statistics the window oracle of its shard alone,
its columns the oracle's at the end; afterwards every rank's P must be the last tick's second.

usage: run_gather_catch_up.py <world> <idx_bytes> <records in total> <config> <closed 0|1>
Prints "ok ..." and exits 0 on success."""
import ctypes as C
import importlib
import os
import sys
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools", "amgen"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
abi = importlib.import_module("active-monitor_b200._lib")
assert "emu" in os.path.basename(abi.LIB_PATH), "run with AMSWEEP_LIB pointing at libamsweep_emu.so"
am = importlib.import_module("active-monitor_b200")
gather = importlib.import_module("active-monitor_b200.gather")
lib = abi.load()

import amgen  # noqa: E402
import window_oracle  # noqa: E402
from adversarial import ZoneMap, product_lookup  # noqa: E402

world, idx_bytes, n_total, config, closed = (int(a) for a in sys.argv[1:6])
mode = abi.SWEEP_CLOSED_LOOP if closed else 0
SEED = 5
T0 = 1790898290  # 2026-10-01 23:44:50 UTC
TICKS = [(T0, False),                    # plain: sets P
         (T0 + 9, True),                 # (23:44:50, 23:44:59]: no minute start, the plain sweep
         (T0 + 9 + 61, True),            # crosses 23:45:00 and 23:46:00
         (T0 + 70 + 3607, True),         # an hour, across midnight
         (T0 + 3677 + 86400, True)]      # a whole day

zmap = ZoneMap(product_lookup(lib))  # zone ids in the generator's order, before anything is classified
whole = amgen.fill(config, 4, 0, n_total, T0, lib.am_healthcheck_classify, threads=2)
shards = [gather.shard_range(n_total, r, world) for r in range(world)]
bases = np.array([s[0] for s in shards], dtype=np.uint64)
sizes = np.array([s[1] for s in shards], dtype=np.uint64)


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


ocols_whole = {k: v.copy() for k, v in whole.items()}
want = oracle_run(ocols_whole, 0)
shard_want, shard_cols = [], []
for first, cnt in shards:
    oc = {k: v[first:first + cnt].copy() for k, v in whole.items()}
    shard_want.append(oracle_run(oc, first))
    shard_cols.append(oc)
handles = [None] * world
errors = []
bar = threading.Barrier(world)


def view(ptr, n, ctype, dtype):
    if n == 0:
        return np.zeros(0, dtype)
    return np.frombuffer((ctype * n).from_address(ptr), dtype=dtype).copy()


def rank_main(rank):
    try:
        first, cnt = shards[rank]
        s = am.Sweep(capacity=cnt, device=rank, shard_base=first)
        s.load_range(0, {k: np.ascontiguousarray(v[first:first + cnt]) for k, v in whole.items()})
        s.set_seed(SEED)
        h = C.c_void_p()
        assert lib.am_gather_create(C.byref(h), rank, rank, world, n_total, idx_bytes) == 0
        mine = C.create_string_buffer(abi.IPC_HANDLE_BYTES)
        assert lib.am_gather_export(h, mine) == 0
        handles[rank] = bytes(mine.raw)
        bar.wait()
        assert lib.am_gather_connect(h, b"".join(handles)) == 0
        assert lib.am_gather_set_layout(h, bases.ctypes.data, sizes.ctypes.data) == 0
        assert lib.am_gather_bind(h, s._h, None, None) == 0
        st = np.zeros(1, dtype=abi.STATS_DTYPE)
        it, dt = (C.c_uint32, np.uint32) if idx_bytes == 4 else (C.c_uint64, np.uint64)
        for k, (T, catch_up) in enumerate(TICKS):
            v = abi.AmTickView()
            m = mode | (abi.SWEEP_CATCH_UP if catch_up else 0)
            rc = lib.am_gather_tick_view(h, T, m, C.byref(v), C.cast(st.ctypes.data, C.POINTER(abi.AmTickStats)))
            assert rc == 0, (rc, lib.am_gather_last_error(h))
            counts = view(lib.am_gather_out_counts(h), world + 1, C.c_uint32, np.uint32)
            total = int(counts[world])
            gi = view(lib.am_gather_out_idx(h), total, it, dt).astype(np.uint64)
            ga = view(lib.am_gather_out_act(h), total, C.c_uint8, np.uint8)
            wi, wa, _ = want[k]
            np.testing.assert_array_equal(gi, wi, err_msg=f"rank {rank} tick {k} idx")
            np.testing.assert_array_equal(ga.astype(np.uint32), wa, err_msg=f"rank {rank} tick {k} act")
            oi, oa, ost = shard_want[rank][k]
            got = {f: int(st[f][0]) for f in abi.STAT_FIELDS}
            assert got == ost, (rank, k, got, ost)
            vi = view(C.cast(v.idx_local, C.c_void_p).value, int(v.n), C.c_uint32, np.uint32)
            va = view(C.cast(v.action, C.c_void_p).value, int(v.n), C.c_uint8, np.uint8)
            np.testing.assert_array_equal(vi.astype(np.uint64) + np.uint64(first), oi, err_msg=f"rank {rank} tick {k} view")
            np.testing.assert_array_equal(va.astype(np.uint32), oa, err_msg=f"rank {rank} tick {k} view act")
        bar.wait()
        dev = s.read_range(0, cnt)
        for name in abi.COLUMN_NAMES:
            np.testing.assert_array_equal(dev[name], shard_cols[rank][name], err_msg=f"rank {rank} column {name}")
        # P is the last tick's second on every rank: a day and a second later is refused, without effect (no exchange
        # needed), a day later is accepted
        last = TICKS[-1][0]
        rc = lib.am_sweep_tick_shard(s._h, last + 86401, mode | abi.SWEEP_CATCH_UP, None)
        assert rc == abi.AM_E_RANGE, (rank, rc)
        rc = lib.am_sweep_tick_shard(s._h, last + 86400, mode | abi.SWEEP_CATCH_UP, None)
        assert rc == 0, (rank, rc)
        bar.wait()
        lib.am_gather_destroy(h)
        s.close()
    except BaseException as e:  # noqa: BLE001
        import traceback
        errors.append((rank, repr(e), traceback.format_exc()[-1500:]))
        try:
            bar.abort()
        except Exception:
            pass


th = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
for t in th:
    t.start()
for t in th:
    t.join()
if errors:
    print("FAILED", errors)
    sys.exit(1)
print(f"ok catch-up world={world} idx_bytes={idx_bytes} n={n_total} config={config} closed={closed} "
      f"emitted={[len(w[0]) for w in want]}")
