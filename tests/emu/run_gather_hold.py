"""Child process of tests/test_in_flight_exchange_emulator.py: ticks with the hold in flight on, through the sharded
whole step.  `world` ranks as Python threads drive the REAL C-ABI of the emulated library, as run_gather_catch_up.py
does: every rank owns an index-range shard of ONE amgen population, turns the hold on and calls am_gather_tick_view
(am_sweep_tick_shard, the hold variants, then the exchange).  Ticks at consecutive seconds, across minutes and with
catch-up windows; between them Succeeded / Failed phases are posted for some of the checks in flight, each to the rank
that owns it.  Every rank's global list must equal the hold oracle (tests/hold_oracle.py) of the UNSHARDED population,
its view the part of that list it owns; at the end its columns and am_sweep_in_flight the oracle's.

usage: run_gather_hold.py <world> <idx_bytes> <records in total> <config>
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
from handle_model import NONE, HandleModel  # noqa: E402

world, idx_bytes, n_total, config = (int(a) for a in sys.argv[1:5])
T0 = 1790898290  # 2026-10-01 23:44:50 UTC
TICKS = [(T0, False), (T0 + 1, False), (T0 + 2, False), (T0 + 9, True), (T0 + 70, True), (T0 + 71, False),
         (T0 + 72, False), (T0 + 700, True), (T0 + 701, False), (T0 + 3700, True), (T0 + 3701, False)]

zmap = ZoneMap(product_lookup(lib))  # zone ids in the generator's order, before anything is classified
whole = amgen.fill(config, 4, 0, n_total, T0, lib.am_healthcheck_classify, threads=2)
shards = [gather.shard_range(n_total, r, world) for r in range(world)]
bases = np.array([s[0] for s in shards], dtype=np.uint64)
sizes = np.array([s[1] for s in shards], dtype=np.uint64)

# the model run first: it decides which in-flight checks post a phase before each tick
rng = np.random.default_rng(world * 1000 + config)
model = HandleModel(zmap, n_total, hold=True)
model.load(0, whole)
want, posts = [], []
for k, (T, catch_up) in enumerate(TICKS):
    fl = np.flatnonzero(model.since != NONE)
    sl = np.sort(rng.choice(fl, min(len(fl), 300), replace=False)) if k and len(fl) else np.zeros(0, np.int64)
    ph = rng.integers(1, 3, len(sl)).astype(np.uint8)
    model.post(sl, ph)
    posts.append((sl, ph))
    want.append(model.tick(T, abi.SWEEP_CATCH_UP if catch_up else 0))
assert sum(int(((w[1] & abi.ACT_SUBMIT_HC) != 0).sum()) for w in want[1:]) > 0

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
        s.set_hold_in_flight(True)
        s.load_range(0, {k: np.ascontiguousarray(v[first:first + cnt]) for k, v in whole.items()})
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
            sl, ph = posts[k]
            own = (sl >= first) & (sl < first + cnt)
            if own.any():
                s.post_result(sl[own] - first, ph[own])
            v = abi.AmTickView()
            rc = lib.am_gather_tick_view(h, T, abi.SWEEP_CATCH_UP if catch_up else 0, C.byref(v),
                                         C.cast(st.ctypes.data, C.POINTER(abi.AmTickStats)))
            assert rc == 0, (rc, lib.am_gather_last_error(h))
            counts = view(lib.am_gather_out_counts(h), world + 1, C.c_uint32, np.uint32)
            total = int(counts[world])
            gi = view(lib.am_gather_out_idx(h), total, it, dt).astype(np.uint64)
            ga = view(lib.am_gather_out_act(h), total, C.c_uint8, np.uint8)
            wi, wa = want[k][:2]
            np.testing.assert_array_equal(gi, wi, err_msg=f"rank {rank} tick {k} idx")
            np.testing.assert_array_equal(ga.astype(np.uint32), wa, err_msg=f"rank {rank} tick {k} act")
            part = (wi >= first) & (wi < first + cnt)
            vi = view(C.cast(v.idx_local, C.c_void_p).value, int(v.n), C.c_uint32, np.uint32)
            va = view(C.cast(v.action, C.c_void_p).value, int(v.n), C.c_uint8, np.uint8)
            np.testing.assert_array_equal(vi.astype(np.uint64) + np.uint64(first), wi[part], err_msg=f"rank {rank} tick {k} view")
            np.testing.assert_array_equal(va.astype(np.uint32), wa[part], err_msg=f"rank {rank} tick {k} view act")
        bar.wait()
        dev = s.read_range(0, cnt)
        for name in abi.COLUMN_NAMES:
            np.testing.assert_array_equal(dev[name], model.cols()[name][first:first + cnt], err_msg=f"rank {rank} column {name}")
        np.testing.assert_array_equal(s.in_flight(0, cnt), model.in_flight()[first:first + cnt],
                                      err_msg=f"rank {rank} in_flight")
        # a closed-loop step is refused on every rank before anything happens (no exchange needed)
        rc = lib.am_sweep_tick_shard(s._h, TICKS[-1][0] + 1, abi.SWEEP_CLOSED_LOOP, None)
        assert rc == abi.AM_E_INVAL, (rank, rc)
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
print(f"ok hold world={world} idx_bytes={idx_bytes} n={n_total} config={config} "
      f"emitted={[len(w[0]) for w in want]} held={int((model.since != NONE).sum())}")
