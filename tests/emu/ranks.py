"""The rank harness of the emulator's multi-rank runners (tests/emu/run_gather_*.py).  `world` ranks as Python threads
drive the REAL C-ABI of the emulated library (csrc/sweep.cu + csrc/gather.cu host code, the tick and exchange kernels
on cuda_emu.h; CUDA IPC handles carry plain pointers, cuda_rt_emu.h).  ctypes releases the GIL during a call, so the
ranks' push kernels really run concurrently and meet through their flags.

A runner imports this module first: it puts the repository, the oracle, the generator and the tests on sys.path and
loads the library AMSWEEP_LIB points at, which must be libamsweep_emu.so."""
import ctypes as C
import importlib
import os
import sys
import threading
import traceback

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

T0 = 1790898290  # 2026-10-01 23:44:50 UTC
CATCH_UP = abi.SWEEP_CATCH_UP
# (T, mode): consecutive seconds, minutes crossed by plain ticks and catch-up windows of seconds, minutes and an hour
HOLD_TICKS = [(T0, 0), (T0 + 1, 0), (T0 + 2, 0), (T0 + 9, CATCH_UP), (T0 + 70, CATCH_UP), (T0 + 71, 0), (T0 + 72, 0),
              (T0 + 700, CATCH_UP), (T0 + 701, 0), (T0 + 3700, CATCH_UP), (T0 + 3701, 0)]
CHANGE_TICKS = [(T0, 0), (T0 + 1, 0), (T0 + 10, CATCH_UP), (T0 + 70, CATCH_UP), (T0 + 71, 0), (T0 + 700, CATCH_UP),
                (T0 + 3700, CATCH_UP), (T0 + 3701, 0)]


def population(n_total, config, remedy=False):
    """(zone map, amgen population `config` of n_total records classified by the emulated library).  The map comes
    first: it introduces the zones in the generator's order.  `remedy`: a remedy workflow on half of the records."""
    zmap = ZoneMap(product_lookup(lib))
    whole = amgen.fill(config, 4, 0, n_total, T0, lib.am_healthcheck_classify, threads=2)
    if remedy:
        whole["flags"] |= np.where(np.random.default_rng(config).random(n_total) < 0.5, abi.F_HAS_REMEDY, 0).astype(np.uint32)
    return zmap, whole


def view(ptr, n, ctype, dtype):
    """numpy copy of n elements at a raw address (np.ctypeslib.as_array on a POINTER patches the
    ctypes type object: not safe from several rank threads at once)"""
    if n == 0:
        return np.zeros(0, dtype)
    return np.frombuffer((ctype * n).from_address(ptr), dtype=dtype).copy()


class Shards:
    """the index-range shard of every rank when `world` ranks share n_total records"""

    def __init__(self, n_total, world):
        self.n_total = n_total
        self.shards = [gather.shard_range(n_total, r, world) for r in range(world)]
        self.bases = np.array([s[0] for s in self.shards], dtype=np.uint64)
        self.sizes = np.array([s[1] for s in self.shards], dtype=np.uint64)

    def own(self, slots, rank):
        """mask of the global slots that `rank` owns"""
        first, cnt = self.shards[rank]
        return (slots >= first) & (slots < first + cnt)

    def part(self, cols, rank):
        """a copy of the rows of `rank`'s shard"""
        first, cnt = self.shards[rank]
        return {k: v[first:first + cnt].copy() for k, v in cols.items()}


_exported = {}  # rank -> its IPC handles, read by every rank once all have met at the barrier


class Gather:
    """one rank's gather handle: created and exported, then connected once every rank has exported.  The layout and
    the bound sweep are separate calls, as a rank may check what is refused before either."""

    def __init__(self, rank, bar, cap_total, idx_bytes):
        self.rank, self.world, self.cap_total, self.idx_bytes = rank, bar.parties, cap_total, idx_bytes
        self.h = C.c_void_p()
        assert lib.am_gather_create(C.byref(self.h), rank, rank, self.world, cap_total, idx_bytes) == 0
        mine = C.create_string_buffer(abi.IPC_HANDLE_BYTES)
        assert lib.am_gather_export(self.h, mine) == 0
        _exported[rank] = bytes(mine.raw)
        bar.wait()
        assert lib.am_gather_connect(self.h, b"".join(_exported[r] for r in range(self.world))) == 0
        self.st = np.zeros(1, dtype=abi.STATS_DTYPE)  # this shard's statistics of the last step

    @classmethod
    def bound(cls, rank, bar, shards, s, idx_bytes):
        """connected, laid out as `shards` and bound to the rank's sweep `s`"""
        g = cls(rank, bar, shards.n_total, idx_bytes)
        g.set_layout(shards)
        g.bind(s)
        return g

    def close(self, bar, s=None):
        """once every rank is done with the others' buffers: destroy the handle, and close the sweep `s`"""
        bar.wait()
        lib.am_gather_destroy(self.h)
        if s is not None:
            s.close()

    def set_layout(self, shards):
        assert lib.am_gather_set_layout(self.h, shards.bases.ctypes.data, shards.sizes.ctypes.data) == 0
        self.first = shards.shards[self.rank][0]

    def bind(self, s):
        assert lib.am_gather_bind(self.h, s._h, None, None) == 0

    def counts(self):
        return view(lib.am_gather_out_counts(self.h), self.world + 1, C.c_uint32, np.uint32)

    def read(self):
        """the global (idx, act) lists, idx at the gather's index width, and the counts"""
        counts = self.counts()
        total = int(counts[self.world])
        assert total <= self.cap_total, (self.rank, counts.tolist())
        it, dt = (C.c_uint32, np.uint32) if self.idx_bytes == 4 else (C.c_uint64, np.uint64)
        gi = view(lib.am_gather_out_idx(self.h), total, it, dt).astype(np.uint64)
        ga = view(lib.am_gather_out_act(self.h), total, C.c_uint8, np.uint8)
        return gi, ga, counts

    def tick_view(self, T, mode):
        v = abi.AmTickView()
        rc = lib.am_gather_tick_view(self.h, T, mode, C.byref(v), C.cast(self.st.ctypes.data, C.POINTER(abi.AmTickStats)))
        return rc, v

    def step(self, T, mode):
        """the whole step (am_gather_tick_view) at (T, mode): read() and this rank's view (idx, act), idx global"""
        rc, v = self.tick_view(T, mode)
        assert rc == 0, (rc, lib.am_gather_last_error(self.h))
        gi, ga, counts = self.read()
        assert int(v.shard_base) == self.first, (self.rank, int(v.shard_base))
        vi = view(C.cast(v.idx_local, C.c_void_p).value, int(v.n), C.c_uint32, np.uint32).astype(np.uint64)
        va = view(C.cast(v.action, C.c_void_p).value, int(v.n), C.c_uint8, np.uint8)
        return gi, ga, counts, (vi + np.uint64(self.first), va)


def check_list(rank, k, gi, ga, wi, wa):
    np.testing.assert_array_equal(gi, wi, err_msg=f"rank {rank} tick {k} idx")
    np.testing.assert_array_equal(ga.astype(np.uint32), wa, err_msg=f"rank {rank} tick {k} act")


def check_view(rank, k, vw, wi, wa):
    np.testing.assert_array_equal(vw[0], wi, err_msg=f"rank {rank} tick {k} view")
    np.testing.assert_array_equal(vw[1].astype(np.uint32), wa, err_msg=f"rank {rank} tick {k} view act")


def check_columns(rank, s, want):
    """the sweep's columns equal `want`, its shard's rows"""
    dev = s.read_range(0, len(want["flags"]))
    for name in abi.COLUMN_NAMES:
        np.testing.assert_array_equal(dev[name], want[name], err_msg=f"rank {rank} column {name}")


def run_ranks(world, rank_main):
    """rank_main(rank, barrier) on `world` threads.  A rank that raises breaks the barrier, so no other rank waits for
    it; then the run prints FAILED with every failed rank's error and the tail of its traceback, and exits 1."""
    bar = threading.Barrier(world)
    errors = []

    def main(rank):
        try:
            rank_main(rank, bar)
        except BaseException as e:  # noqa: BLE001
            errors.append((rank, repr(e), traceback.format_exc()[-1500:]))
            bar.abort()

    th = [threading.Thread(target=main, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    if errors:
        print("FAILED", errors)
        sys.exit(1)
