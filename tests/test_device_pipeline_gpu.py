"""Device-resident ticks as a pipeline issues them: am_sweep_tick_device calls queued on several streams behind
a delay kernel, with staged calls, host ticks and reads between them; posting threads while ticks are in flight;
output buffers shorter than the list; shard bases past 2^32; the exchange of a one-GPU world; and output
pointers that are not aligned for the kernels' stores.

Every tick is compared with the sequential model (tests/handle_model.py): the C oracle's columns with every staged
call applied in call order, each tick the oracle's sweep at its second (a catch-up tick: the window oracle over
(P, T]).  The device work is checked after one synchronisation at the end, so a tick that read a staging area, a zone offset or a
window box before (or after) the host wrote it shows up as a difference.

The stream tests need a GPU.  The misalignment test also runs on the emulated library (AMSWEEP_LIB), with numpy
memory standing in for device memory."""
import calendar
import os
import threading

import numpy as np
import pytest

from adversarial import ZoneMap, population, zones_usable
from handle_model import HandleModel

pytestmark = pytest.mark.gpu

EMULATED = "emu" in os.path.basename(os.environ.get("AMSWEEP_LIB", ""))
needs_streams = pytest.mark.skipif(EMULATED, reason="the emulated library completes every call before it returns")

HOUR = 3600
SEED = 5
T_OCT = 1790812800                                    # 2026-10-01 00:00:00 UTC
T_NOV = calendar.timegm((2026, 11, 1, 4, 0, 0))       # St. John's leaves summer time at 04:30 UTC, New York at 06:00
GATE_S = 0.2                                          # the delay kernel that holds the first stream
GUARD = 64                                            # canary entries past every list buffer
C_IDX, C_ACT, C_CNT, C_ST = 0x5A, 0xA5, 0x7E, 0x3C    # canary bytes
U64 = (1 << 64) - 1


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def _sync():
    if not EMULATED:
        import torch
        torch.cuda.synchronize()


def _region(nbytes, fill, offset):
    """`nbytes` of device memory at `offset` bytes past a 256-B boundary, every byte `fill`"""
    if EMULATED:  # the emulated library's device memory is host memory
        a = np.full(nbytes + 512, fill, np.uint8)
        base = a.ctypes.data
    else:
        import torch
        a = torch.full((nbytes + 512,), fill, dtype=torch.uint8, device="cuda")
        base = a.data_ptr()
    skip = (-base) % 256 + offset
    return a, skip, base + skip, nbytes


class DevOut:
    """One set of am_sweep_tick_device outputs, canaries throughout: `cap` list entries and GUARD more, the
    count, the statistics and one more u64.  Offsets misalign the arrays."""

    def __init__(self, cap, offsets=(0, 0, 0, 0)):
        self.cap = cap
        self.r = [_region(b, f, o) for b, f, o in zip(((cap + GUARD) * 4, cap + GUARD, 4, 17 * 8),
                                                      (C_IDX, C_ACT, C_CNT, C_ST), offsets)]

    def args(self, count=True, stats=True):
        """(d_idx, d_act, cap, d_count, d_stats) for Sweep.tick_device; NULL list buffers when cap == 0"""
        p = [r[2] for r in self.r]
        return (p[0] if self.cap else 0, p[1] if self.cap else 0, self.cap, p[2] if count else 0,
                p[3] if stats else 0)

    def fetch(self):
        """(u32 idx, u8 act, count bytes, u64 stats) after the device work has finished"""
        out = []
        for a, skip, _, nb in self.r:
            h = a if EMULATED else a.cpu().numpy()
            out.append(np.ascontiguousarray(h[skip: skip + nb]))
        return out[0].view(np.uint32), out[1], out[2], out[3].view(np.uint64)

    def untouched(self):
        idx, act, cnt, st = self.fetch()
        return (idx == C_IDX * 0x01010101).all() and (act == C_ACT).all() and (cnt == C_CNT).all() and \
            (st == C_ST * 0x0101010101010101).all()


def _stats(am, words):
    return dict(zip(am.abi.STAT_FIELDS, [int(v) & U64 for v in words[:16]]))


def check_device_tick(am, out, want, base, what, count=True, stats=True):
    """the list prefix, the count, the full statistics; canaries everywhere nothing was to be written"""
    wi, wa, ws = want[:3]
    idx, act, cnt, st = out.fetch()
    m = min(len(wi), out.cap)
    if count:
        assert int(cnt.view(np.uint32)[0]) == m, (what, "count", int(cnt.view(np.uint32)[0]), m, len(wi))
    else:
        assert (cnt == C_CNT).all(), (what, "count written")
    np.testing.assert_array_equal(idx[:m].astype(np.uint64) + np.uint64(base), wi[:m], err_msg=f"{what}: idx")
    np.testing.assert_array_equal(act[:m].astype(np.uint32), wa[:m], err_msg=f"{what}: act")
    assert (idx[m:] == C_IDX * 0x01010101).all(), (what, "idx past the list", int(np.flatnonzero(idx[m:] != C_IDX * 0x01010101)[0]) + m)
    assert (act[m:] == C_ACT).all(), (what, "act past the list", int(np.flatnonzero(act[m:] != C_ACT)[0]) + m)
    if stats:
        got = _stats(am, st)
        assert got == ws, (what, {f: (got[f], ws[f]) for f in ws if got[f] != ws[f]})
    else:
        assert (st[:16] == C_ST * 0x0101010101010101).all(), (what, "stats written")
    assert int(st[16]) == C_ST * 0x0101010101010101, (what, "past the statistics")


def check_host_tick(got, want, what):
    gi, ga, gs = got
    wi, wa, ws = want[:3]
    assert gs == ws, (what, {f: (gs[f], ws[f]) for f in ws if gs[f] != ws[f]})
    np.testing.assert_array_equal(np.asarray(gi, np.uint64), wi, err_msg=f"{what}: idx")
    np.testing.assert_array_equal(np.asarray(ga, np.uint32), wa, err_msg=f"{what}: act")


def check_columns(am, dev, model, what):
    """flags everywhere; the other columns of live slots (a removed slot keeps only its tombstone)"""
    np.testing.assert_array_equal(dev["flags"], model["flags"], err_msg=f"{what}: flags")
    live = (model["flags"] & np.uint32(am.F_TOMBSTONE)) == 0
    for name in am.COLUMN_NAMES:
        np.testing.assert_array_equal(dev[name][live], model[name][live], err_msg=f"{what}: {name}")


def _model(zmap, cols, base=0):
    """the model of a handle without the hold, `cols` loaded into slots 0.."""
    m = HandleModel(zmap, len(cols["flags"]), base, seed=SEED)
    m.load(0, cols)
    return m


def _results(rng, n, every, offset=None):
    """a post_result pair (workflow phases, then remedy phases) on every `every`-th slot"""
    slots = np.arange(int(rng.integers(0, every)) if offset is None else offset, n, every, dtype=np.uint64)
    phase = rng.integers(1, 3, len(slots)).astype(np.uint8)
    rphase = rng.integers(0, 3, len(slots)).astype(np.uint8)
    return [("post", slots, phase, None), ("post", slots, np.zeros_like(phase), rphase)]


def _apply(s, model, op):
    """a staged call on the library (model None) or on the model (s None)"""
    kind, idx = op[0], op[1]
    if s is not None:
        {"post": lambda: s.post_result(idx, op[2], op[3]), "upsert": lambda: s.upsert(idx, op[2]),
         "remove": lambda: s.remove(idx)}[kind]()
    else:
        idx = idx.astype(np.int64)
        {"post": lambda: model.post(idx, op[2], op[3]), "upsert": lambda: model.upsert(idx, op[2]),
         "remove": lambda: model.remove(idx)}[kind]()


def _both(s, model, ops):
    for op in ops:
        _apply(s, None, op)
        _apply(None, model, op)


def _gate(torch, stream):
    """a delay kernel of about GATE_S on `stream` (it ends by itself); returns an event recorded behind it"""
    done = torch.cuda.Event()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(GATE_S * 2.0e9))  # clock cycles; the H100 runs its SMs at up to 1.98 GHz
        done.record(stream)
    return done


# ---- 1. a queued sequence of device ticks on four streams, staged work between them ----------------------------
@needs_streams
def test_queued_ticks_on_four_streams_equal_the_oracle_sequence(am, zmap):
    """Two gated phases.  In the first, two catch-up ticks in a row queue their window boxes while the gate holds
    the stream: the second must not overwrite the pinned boxes before the first copy has left them.  In the
    second, two ticks cross an offset change of a registered zone (St. John's, then New York) and refresh the
    zone offsets the same way."""
    import torch
    n = 100_003
    rng = np.random.default_rng(101)
    tz_ids = zmap.ids_of(zones_usable(T_NOV - HOUR, T_NOV + 3 * HOUR))
    cols = population(rng, n, T_NOV, True, tz_ids)
    model = _model(zmap, cols)

    def fresh(k):
        idx = rng.choice(n, k, replace=False).astype(np.uint64)
        return idx, am.columns_to_records(population(rng, k, T_NOV, True, tz_ids))

    def removes(k):
        return ("remove", rng.choice(n, k, replace=False).astype(np.uint64))

    # a UTC-bound 5-field record, bound to St. John's and back by two upserts
    f0 = cols["flags"]
    j = int(np.flatnonzero(((f0 & 7) == am.KIND_CRON_SPEC) & ((f0 >> 24) == 0) & ((f0 & am.F_TOMBSTONE) == 0))[0])
    to_zone = am.columns_to_records({k: v[j:j + 1].copy() for k, v in cols.items()})
    to_zone["flags"] |= np.uint32(zmap.ids["America/St_Johns"] << 24)
    to_utc = to_zone.copy()
    to_utc["flags"] &= np.uint32(0x00FFFFFF)
    CU, CL, FS = am.SWEEP_CATCH_UP, am.SWEEP_CLOSED_LOOP, am.SWEEP_FULL_SCAN
    M = 60
    seq = (
        [("gate",), ("dev", T_NOV, 0, "A")] + _results(rng, n, 23) +
        [("dev", T_NOV + 13, CL, "own"),
         ("dev", T_NOV + M + 15, CU | CL, "B"),                           # (04:00:13, 04:01:15]
         ("dev", T_NOV + 2 * M + 10, CU | FS, "null")] +                  # (04:01:15, 04:02:10]: other boxes
        _results(rng, n, 2) + [("upsert",) + fresh(40), removes(30)] +
        [("dev", T_NOV + 3 * M, CL, "own")] +
        _results(rng, n, 2) + [("upsert", np.array([j], np.uint64), to_zone)] +  # the same area again: early chunks
        [("host", T_NOV + 3 * M + 30, 0)] + _results(rng, n, 1, 0) +            # the staging arrays grow
        [("dev", T_NOV + 4 * M, FS | CL, "B"), ("next_due", T_NOV + 4 * M)] + _results(rng, n, 23) +
        [("dev", T_NOV + 4 * M + 20, CU, "null"), ("read",)] +           # no minute start in the window
        [("upsert", np.array([j], np.uint64), to_utc)] + _results(rng, n, 2) + [removes(30), ("upsert",) + fresh(7)] +
        [("gate",), ("dev", T_NOV + 30 * M, 0, "A"),                     # 04:30: St. John's changed its offset
         ("dev", T_NOV + 120 * M, FS, "own")] +                          # 06:00: New York changed its offset
        _results(rng, n, 1, 0) + _results(rng, n, 1, 0) +
        [("dev", T_NOV + 120 * M + 45, CL, "null")] + _results(rng, n, 5) +
        [("dev", T_NOV + 151 * M + 5, CU, "B"), ("dev", T_NOV + 151 * M + 6, CU | CL, "A")]
    )
    outs = {k: DevOut(n) for k, op in enumerate(seq) if op[0] == "dev"}
    A, B = torch.cuda.Stream(), torch.cuda.Stream()
    with am.Sweep(capacity=n) as s:
        s.load_range(0, cols)
        s.set_seed(SEED)
        # a host tick first: the sweep's kernels are loaded before the gate
        check_host_tick(s.tick(T_NOV - HOUR), model.tick(T_NOV - HOUR, 0), "warm-up")
        streams = {"A": A.cuda_stream, "B": B.cuda_stream, "own": s.stream, "null": 0}
        torch.cuda.synchronize()
        seen, pending = {}, []
        for k, op in enumerate(seq):
            if op[0] == "gate":
                gate = _gate(torch, A)
            elif op[0] == "dev":
                s.tick_device(op[1], op[2], *outs[k].args(), stream=streams[op[3]])
            elif op[0] == "host":
                seen[k] = tuple(np.array(v, copy=True) if not isinstance(v, dict) else v for v in s.tick(op[1], op[2]))
            elif op[0] == "next_due":
                seen[k] = s.next_due(op[1])
            elif op[0] == "read":
                seen[k] = s.read_range(0, n)
            else:
                _apply(s, None, op)
            pending.append((k, op[0], not gate.query()))
        torch.cuda.synchronize()
        # the device ticks up to the first that must wait for a copy behind the gate (the second window, the
        # second zone refresh) returned while the gate still held the first stream: queued, not run.  Where a
        # later call waited for the device is printed, not asserted.
        devs = [p for p in pending if p[1] == "dev"]
        assert devs[0][2] and devs[1][2] and devs[2][2] and devs[7][2], pending
        print("gate still running after:", [(k, kind) for k, kind, p in pending if p])
        for k, op in enumerate(seq):
            what = (k, op[0], op[1] if len(op) > 1 and not isinstance(op[1], np.ndarray) else None)
            if op[0] == "gate":
                continue
            if op[0] == "dev":
                check_device_tick(am, outs[k], model.tick(op[1], op[2]), 0, what)
            elif op[0] == "host":
                check_host_tick(seen[k], model.tick(op[1], op[2]), what)
            elif op[0] == "next_due":
                assert seen[k] == model.first_active_tick(op[1], 120), what
            elif op[0] == "read":
                check_columns(am, seen[k], model.cols(), what)
            else:
                _apply(None, model, op)
        check_columns(am, s.read_range(0, n), model.cols(), "final")


# ---- 2. posting threads between device ticks that are still in flight -------------------------------------------
@needs_streams
def test_posting_threads_between_queued_device_ticks(am, zmap):
    import torch
    n = 100_003
    T0 = T_OCT + 14 * HOUR
    rng = np.random.default_rng(202)
    tz_ids = zmap.ids_of(zones_usable(T0, T0 + HOUR))
    cols = population(rng, n, T0, True, tz_ids)
    model = _model(zmap, cols)
    up_slots = np.arange(3, n, 97, dtype=np.uint64)              # the upserting thread's slots
    free = np.setdiff1d(np.arange(n, dtype=np.uint64), up_slots)
    lanes = [free[w::4] for w in range(4)]                        # four posting threads, disjoint slots
    CU, CL, FS = am.SWEEP_CATCH_UP, am.SWEEP_CLOSED_LOOP, am.SWEEP_FULL_SCAN
    # Two rounds before the gate bring both staging areas to the size of a round: growing a staging array frees
    # the old pinned or device array, and freeing memory waits for the device.
    WARM = 2
    ticks = [(T0 - 120, 0), (T0 - 60, CL)] + \
        [(T0, 0), (T0 + 7, CL), (T0 + 60, FS), (T0 + 200, CU | CL), (T0 + 201, 0), (T0 + 1500, CU), (T0 + 1560, CL)]
    rounds = []
    for _ in ticks:
        posts = []
        for lane in lanes:
            calls = []
            for dense in (False, True, False):
                sl = rng.choice(lane, len(lane) // (1 if dense else 11), replace=False)
                calls.append((sl, rng.integers(0, 3, len(sl)).astype(np.uint8),
                              rng.integers(0, 3, len(sl)).astype(np.uint8) if rng.integers(0, 2) else None))
            posts.append(calls)
        ups = [(u, am.columns_to_records(population(rng, len(u), T0, True, tz_ids)))
               for u in (rng.choice(up_slots, 50, replace=False), rng.choice(up_slots, 50, replace=False))]
        rounds.append((posts, ups))
    outs = [DevOut(n) for _ in ticks]
    A, B = torch.cuda.Stream(), torch.cuda.Stream()
    with am.Sweep(capacity=n) as s:
        s.load_range(0, cols)
        s.set_seed(SEED)
        check_host_tick(s.tick(T0 - 180), model.tick(T0 - 180, 0), "warm-up")
        streams = [A.cuda_stream, s.stream, B.cuda_stream, 0]
        errors, pending = [], []

        def run(fn):
            try:
                fn()
            except Exception as e:  # reported by the ticking thread
                errors.append(e)

        gate = None
        for k, ((T, mode), (posts, ups)) in enumerate(zip(ticks, rounds)):
            if k == WARM:
                torch.cuda.synchronize()
                gate = _gate(torch, A)
            th = [threading.Thread(target=run, args=(lambda c=calls: [s.post_result(*x) for x in c],)) for calls in posts]
            th.append(threading.Thread(target=run, args=(lambda: [s.upsert(u, r) for u, r in ups],)))
            for t in th:
                t.start()
            for t in th:
                t.join()
            assert not errors, errors
            s.tick_device(T, mode, *outs[k].args(), stream=streams[k % 4])
            pending.append(gate is not None and not gate.query())
        torch.cuda.synchronize()
        assert pending[WARM], pending
        print("gate still running after ticks:", [k for k, p in enumerate(pending) if p])
        for k, ((T, mode), (posts, ups)) in enumerate(zip(ticks, rounds)):
            for calls in posts:
                for sl, ph, rp in calls:
                    model.post(sl.astype(np.int64), ph, rp)
            for u, r in ups:
                model.upsert(u.astype(np.int64), r)
            check_device_tick(am, outs[k], model.tick(T, mode), 0, (k, T, mode))
        check_columns(am, s.read_range(0, n), model.cols(), "final")


# ---- 3. device buffers shorter than the list ------------------------------------------------------------------------
def _short_caps(wi_local, n_emitted):
    """1, 3, 4, 5; a cut inside the ragged first quad of a group; a group boundary; around the list's end"""
    caps = {1, 3, 4, 5, 8192, max(n_emitted - 1, 0), n_emitted, n_emitted + 1}
    starts = np.searchsorted(wi_local, np.arange(8192, int(wi_local[-1]) + 1 if len(wi_local) else 0, 8192))
    ends = np.append(starts[1:], n_emitted)
    ragged = [int(a) for a, b in zip(starts, ends) if int(a) % 4 in (1, 2) and b - a >= 2]
    if ragged:
        caps.add(ragged[0] + 1)  # the group's first quad holds entries before and after the cut
    if len(starts):
        caps.add(int(starts[0]))  # the list position of local index 8192
    return sorted(caps), bool(ragged)


@needs_streams
@pytest.mark.parametrize("n", [8193, 100_003])
@pytest.mark.parametrize("how", ["open", "closed", "catch-up"])
def test_short_device_buffers(am, zmap, n, how):
    P = T_OCT + 9 * HOUR + 17
    T = P + (1800 if how == "catch-up" else 43)
    mode = {"open": 0, "closed": am.SWEEP_CLOSED_LOOP, "catch-up": am.SWEEP_CATCH_UP}[how]
    rng = np.random.default_rng(n + len(how))
    cols = population(rng, n, T, True, zmap.ids_of(zones_usable(P, T + 1)))
    staged = _results(rng, n, 23)
    model = _model(zmap, cols)
    want_P = model.tick(P, 0) if how == "catch-up" else None
    for op in staged:
        _apply(None, model, op)
    want = model.tick(T, mode)
    want_next = model.tick(T + 1, mode & am.SWEEP_CLOSED_LOOP)
    n_emitted = len(want[0])
    caps, ragged = _short_caps(want[0].astype(np.int64), n_emitted)
    assert n_emitted > 5 and (ragged or n < 50_000), (n_emitted, caps)
    cases = [(0, True, True)] + [(c, True, True) for c in caps] + [(n_emitted // 2, False, True), (n_emitted, True, False)]
    for cap, count, stats in cases:
        with am.Sweep(capacity=n) as s:
            s.load_range(0, cols)
            s.set_seed(SEED)
            if how == "catch-up":
                check_host_tick(s.tick(P), want_P, "P")
            for op in staged:
                _apply(s, None, op)
            out = DevOut(cap)
            s.tick_device(T, mode, *out.args(count, stats), stream=s.stream)
            _sync()
            check_device_tick(am, out, want, 0, (how, n, cap, count, stats), count, stats)
            # the short tick consumed its one-shot actions like any other: the next one equals the oracle's
            check_host_tick(s.tick(T + 1, mode & am.SWEEP_CLOSED_LOOP), want_next, (how, n, cap, "next"))
            check_columns(am, s.read_range(0, n), model.cols(), (how, n, cap))


# ---- 4. shard bases past 2^32 -----------------------------------------------------------------------------------------
BASES = [(1 << 32) - 8192 * 3 - 5, (1 << 32) - 1, 1 << 32, (1 << 33) + 5, (1 << 40) + 123]


@needs_streams
@pytest.mark.parametrize("base", BASES, ids=hex)
def test_shard_bases_across_2_32(am, zmap, base):
    n = 100_003
    T0 = T_OCT + 14 * HOUR
    rng = np.random.default_rng(base & 0xFFFF)
    cols = population(rng, n, T0, True, zmap.ids_of(zones_usable(T0, T0 + HOUR)))
    model = _model(zmap, cols, base)
    CU, CL = am.SWEEP_CATCH_UP, am.SWEEP_CLOSED_LOOP
    with am.Sweep(capacity=n, shard_base=base) as s:
        s.load_range(0, cols)
        s.set_seed(SEED)
        check_host_tick(s.tick(T0), model.tick(T0, 0), "tick")
        post = _results(rng, n, 23)
        _both(s, model, post)
        vi, va, vs = s.tick_view(T0 + 1, CL)
        check_host_tick((vi.astype(np.uint64) + np.uint64(base), va, vs), model.tick(T0 + 1, CL), "tick_view")
        full = DevOut(n)
        s.tick_device(T0 + 60, 0, *full.args(), stream=s.stream)
        _sync()
        check_device_tick(am, full, model.tick(T0 + 60, 0), base, "tick_device")
        want = model.tick(T0 + 61, CL)
        short = DevOut(len(want[0]) // 2 + 1)
        s.tick_device(T0 + 61, CL, *short.args(), stream=s.stream)
        _sync()
        check_device_tick(am, short, want, base, "tick_device short")
        _both(s, model, post)
        check_host_tick(s.tick(T0 + 61 + 900, CU | CL), model.tick(T0 + 61 + 900, CU | CL), "catch-up")
        for blocked in (0, am.SWEEP_BLOCKED):
            _both(s, model, post)
            t0 = model.P + 1
            rows = s.run_ticks(t0, 5, mode=CL | blocked, seed=SEED)
            for k in range(5):
                got = {f: int(rows[k][f]) for f in am.abi.STAT_FIELDS}
                ws = model.tick(t0 + k, CL)[2]
                assert got == ws, (blocked, k, {f: (got[f], ws[f]) for f in ws if got[f] != ws[f]})
        check_columns(am, s.read_range(0, n), model.cols(), "final")


# ---- 5. the exchange of a one-GPU world ------------------------------------------------------------------------------
@needs_streams
@pytest.mark.parametrize("idx_bytes,base", [(8, (1 << 33) + 5), (4, (1 << 32) - 100_003 - 3)], ids=["u64", "u32"])
def test_exchange_of_a_one_gpu_world(am, zmap, idx_bytes, base):
    import torch
    gather = __import__("importlib").import_module("active-monitor_b200.gather")
    n = 100_003
    T0 = T_OCT + 16 * HOUR
    rng = np.random.default_rng(idx_bytes)
    cols = population(rng, n, T0, True, zmap.ids_of(zones_usable(T0, T0 + HOUR)))
    model = _model(zmap, cols, base)
    CU, CL, FS = am.SWEEP_CATCH_UP, am.SWEEP_CLOSED_LOOP, am.SWEEP_FULL_SCAN
    # two steps before the gate: the exchange's kernels are loaded and both staging areas have their size
    WARM = 2
    ticks = [(T0 - 60, 0), (T0, CL)] + \
        [(T0 + 1, 0), (T0 + 2, CL), (T0 + 400, CU), (T0 + 401, FS), (T0 + 1300, CU | CL), (T0 + 1320, 0)]
    posts = [_results(rng, n, 23) for _ in ticks]
    idt = torch.int64 if idx_bytes == 8 else torch.int32
    dev = torch.device("cuda:0")
    got_idx = [torch.full((n,), -1, dtype=idt, device=dev) for _ in ticks]
    got_act = [torch.full((n,), C_ACT, dtype=torch.uint8, device=dev) for _ in ticks]
    got_cnt = [torch.full((2,), -1, dtype=torch.int32, device=dev) for _ in ticks]
    got_st = [torch.full((16,), -1, dtype=torch.int64, device=dev) for _ in ticks]
    A, B = torch.cuda.Stream(), torch.cuda.Stream()
    with am.Sweep(capacity=n, shard_base=base) as s:
        s.load_range(0, cols)
        s.set_seed(SEED)
        g = gather.PeerGather(0, cap_total=n, idx_bytes=idx_bytes, shard=(base, n))
        try:
            pending, gate = [], None
            for k, (T, mode) in enumerate(ticks):
                if k == WARM:
                    torch.cuda.synchronize()
                    gate = _gate(torch, A)
                for op in posts[k]:
                    _apply(s, None, op)
                s.tick_shard(T, mode, stream=A.cuda_stream)
                g.exchange(s, got_st[k].data_ptr(), stream=B.cuda_stream)
                idx_v, act_v = g.buffers()  # the output buffers of this exchange's epoch
                with torch.cuda.stream(B):
                    got_idx[k].copy_(idx_v)
                    got_act[k].copy_(act_v)
                    got_cnt[k].copy_(g.counts())
                pending.append(gate is not None and not gate.query())
            torch.cuda.synchronize()
            assert pending[WARM], pending
            print("gate still running after exchanges:", [k for k, p in enumerate(pending) if p])
            mask = (1 << (8 * idx_bytes)) - 1
            for k, (T, mode) in enumerate(ticks):
                for op in posts[k]:
                    _apply(None, model, op)
                wi, wa, ws = model.tick(T, mode)[:3]
                cnt = got_cnt[k].cpu().numpy()
                assert cnt[0] == len(wi) and cnt[1] == len(wi), (k, cnt, len(wi))
                gi = got_idx[k].cpu().numpy()[: len(wi)].astype(np.int64).astype(np.uint64) & np.uint64(mask)
                np.testing.assert_array_equal(gi, wi, err_msg=f"exchange {k}: idx")
                np.testing.assert_array_equal(got_act[k].cpu().numpy()[: len(wi)].astype(np.uint32), wa,
                                              err_msg=f"exchange {k}: act")
                st = _stats(am, got_st[k].cpu().numpy().view(np.uint64))
                assert st == ws, (k, {f: (st[f], ws[f]) for f in ws if st[f] != ws[f]})
            # one step through bind + tick_view: this rank's part of the global list, as local slots
            g.bind(s, A.cuda_stream, B.cuda_stream)
            T = ticks[-1][0] + 60
            vi, va, vs = g.tick_view(T, CU | CL)
            check_host_tick((vi.astype(np.uint64) + np.uint64(base), va, vs), model.tick(T, CU | CL), "tick_view")
            # one through push of a tick_device list
            out = DevOut(n)
            s.tick_device(T + 1, CL, *out.args(), stream=A.cuda_stream)
            d_idx, d_act, _, d_cnt, _ = out.args()
            g.push(d_idx, d_act, d_cnt, base, A.cuda_stream)
            torch.cuda.synchronize()
            want = model.tick(T + 1, CL)
            check_device_tick(am, out, want, base, "tick_device before the push")
            pi, pa, pc = g.result()
            assert pc == [len(want[0])]
            np.testing.assert_array_equal(pi.cpu().numpy().astype(np.int64).astype(np.uint64) & np.uint64(mask), want[0])
            np.testing.assert_array_equal(pa.cpu().numpy().astype(np.uint32), want[1])
            check_columns(am, s.read_range(0, n), model.cols(), "final")
        finally:
            g.close()


@needs_streams
def test_u32_exchange_layout_must_end_at_2_32(am):
    import ctypes as C
    gather = __import__("importlib").import_module("active-monitor_b200.gather")
    g = gather.PeerGather(0, cap_total=64, idx_bytes=4)
    try:
        for base, size, rc in [((1 << 32) - 8, 9, am.AM_E_RANGE), ((1 << 32) - 8, 8, am.AM_OK), (1 << 32, 1, am.AM_E_RANGE)]:
            b = np.array([base], np.uint64)
            z = np.array([size], np.uint64)
            assert g._lib.am_gather_set_layout(g._h, C.c_void_p(b.ctypes.data), C.c_void_p(z.ctypes.data)) == rc, (base, size)
    finally:
        g.close()


# ---- 6. misaligned output pointers (also on the emulated library) ---------------------------------------------------
def test_misaligned_outputs_are_refused_before_anything_happens(am, zmap):
    n = 1023
    P = T_OCT + 11 * HOUR + 29
    T = P + 1800 + 14
    rng = np.random.default_rng(606)
    tz_ids = zmap.ids_of(zones_usable(P, T))
    cols = population(rng, n, P, True, tz_ids)
    model = _model(zmap, cols)
    staged = _results(rng, n, 2) + [("upsert", np.arange(5, 25, dtype=np.uint64),
                                     am.columns_to_records(population(rng, 20, P, True, tz_ids))),
                                    ("remove", np.array([7, 900], np.uint64))] + _results(rng, n, 7)
    CU = am.SWEEP_CATCH_UP
    with am.Sweep(capacity=n) as s:
        s.load_range(0, cols)
        s.set_seed(SEED)
        check_host_tick(s.tick(P), model.tick(P, 0), "P")
        _both(s, model, staged)
        bad =[(4, 0, 0, 0), (8, 0, 0, 0), (12, 0, 0, 0), (1, 0, 0, 0), (0, 1, 0, 0), (0, 2, 0, 0), (0, 0, 2, 0),
               (0, 0, 1, 0), (0, 0, 0, 4), (0, 0, 0, 2)]
        outs = [DevOut(n, off) for off in bad]
        for off, out in zip(bad, outs):
            with pytest.raises(am.AmError) as e:
                s.tick_device(T, CU, *out.args(), stream=s.stream)
            assert e.value.code == am.AM_E_INVAL, off
        _sync()
        for off, out in zip(bad, outs):
            assert out.untouched(), off
        # nothing was drained and P did not move: the aligned tick sees the staged calls and the window (P, T]
        out = DevOut(n)
        s.tick_device(T, CU, *out.args(), stream=s.stream)
        _sync()
        want = model.tick(T, CU)
        assert want[2]["n_result_ok"] + want[2]["n_result_fail"] > 0
        check_device_tick(am, out, want, 0, "aligned")
        check_columns(am, s.read_range(0, n), model.cols(), "final")
