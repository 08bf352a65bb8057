"""Child process of tests/test_status_changes_emulator.py: status changes through the sharded whole step.  `world`
ranks as Python threads drive the REAL C-ABI of the emulated library: every rank owns an index-range shard of ONE amgen
population (half of it with a remedy workflow), turns tracking on, upserts its records and calls am_gather_tick_view
(am_sweep_tick_shard, then the exchange).  Between ticks results are posted, each to the rank that owns its slot (one
tick's batch dense enough for the sweep to apply it), and some ranks read in between.  Every rank's global list must
equal the oracle of the UNSHARDED population, and its am_sweep_last_changes the part of the changed-set oracle
(tests/changes_oracle.py, through tests/handle_model.py) it owns, with the oracle's columns.

usage: run_gather_changes.py <world> <idx_bytes> <records in total> <config>
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
from adversarial import ZoneMap, product_lookup  # noqa: E402
from handle_model import HandleModel  # noqa: E402

world, idx_bytes, n_total, config = (int(a) for a in sys.argv[1:5])
T0 = 1790898290  # 2026-10-01 23:44:50 UTC
TICKS = [(T0, False), (T0 + 1, False), (T0 + 10, True), (T0 + 70, True), (T0 + 71, False), (T0 + 700, True),
         (T0 + 3700, True), (T0 + 3701, False)]

zmap = ZoneMap(product_lookup(lib))  # zone ids in the generator's order, before anything is classified
whole = amgen.fill(config, 4, 0, n_total, T0, lib.am_healthcheck_classify, threads=2)
whole["flags"] |= np.where(np.random.default_rng(config).random(n_total) < 0.5, abi.F_HAS_REMEDY, 0).astype(np.uint32)
shards = [gather.shard_range(n_total, r, world) for r in range(world)]
bases = np.array([s[0] for s in shards], dtype=np.uint64)
sizes = np.array([s[1] for s in shards], dtype=np.uint64)

rng = np.random.default_rng(world * 1000 + config)
model = HandleModel(zmap, n_total, track=True)
model.upsert(np.arange(n_total), am.columns_to_records(whole))
want, posts = [], []
for k, (T, catch_up) in enumerate(TICKS):
    m = n_total // 4 if k == 3 else 200  # tick 3: more than an eighth of the records, applied inside the sweep
    sl = np.sort(rng.choice(n_total, m, replace=False)) if k else np.zeros(0, np.int64)
    ph = rng.integers(0, 3, len(sl)).astype(np.uint8)
    rp = rng.integers(0, 3, len(sl)).astype(np.uint8)
    model.post(sl, ph, rp)
    posts.append((sl, ph, rp))
    out = model.tick(T, abi.SWEEP_CATCH_UP if catch_up else 0)
    want.append((out[0], out[1], model.changes(), {n: model.cols()[n][model.changes()].copy() for n in abi.COLUMN_NAMES}))
assert sum(len(w[2]) for w in want) > n_total // 8

handles = [None] * world
listed = [0] * world
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
        s.set_track_changes(True)
        s.upsert(np.arange(cnt), am.columns_to_records({k: np.ascontiguousarray(v[first:first + cnt]) for k, v in whole.items()}))
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
            sl, ph, rp = posts[k]
            own = (sl >= first) & (sl < first + cnt)
            if own.any():
                s.post_result(sl[own] - first, ph[own], rp[own])
                if (rank + k) % 2:  # a read leaves them pending for the tick
                    s.read(sl[own][:5] - first)
            v = abi.AmTickView()
            rc = lib.am_gather_tick_view(h, T, abi.SWEEP_CATCH_UP if catch_up else 0, C.byref(v),
                                         C.cast(st.ctypes.data, C.POINTER(abi.AmTickStats)))
            assert rc == 0, (rc, lib.am_gather_last_error(h))
            counts = view(lib.am_gather_out_counts(h), world + 1, C.c_uint32, np.uint32)
            total = int(counts[world])
            gi = view(lib.am_gather_out_idx(h), total, it, dt).astype(np.uint64)
            ga = view(lib.am_gather_out_act(h), total, C.c_uint8, np.uint8)
            wi, wa, wc, wcols = want[k]
            np.testing.assert_array_equal(gi, wi, err_msg=f"rank {rank} tick {k} idx")
            np.testing.assert_array_equal(ga.astype(np.uint32), wa, err_msg=f"rank {rank} tick {k} act")
            ci, cc = s.last_changes()
            part = (wc >= first) & (wc < first + cnt)
            np.testing.assert_array_equal(ci, wc[part], err_msg=f"rank {rank} tick {k} changes")
            for name in abi.COLUMN_NAMES:
                np.testing.assert_array_equal(cc[name], wcols[name][part], err_msg=f"rank {rank} tick {k} {name}")
            listed[rank] += len(ci)
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
assert all(v > 0 for v in listed), listed
print(f"ok status changes listed_per_rank={listed} world={world} idx_bytes={idx_bytes} n={n_total} config={config} "
      f"changed={[len(w[2]) for w in want]}")
