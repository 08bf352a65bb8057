"""Checkpoints, delta chains and restores issued while ticks are queued on other streams and while other threads tick,
post and query (include/amsweep.h, "Checkpoint of local slots" and "Delta checkpoints").  A checkpoint holds the tick
guard only while its drain and device passes are issued on the handle's stream; the copy into the caller's buffer and
a delta's commit into the chain's base image follow on the checkpoint stream while ticks go on; a restore uploads and
verifies its blob before it takes the guard.  A missing wait would let a blob capture part of a tick, and a standby
would resume from a state the source never had.

Every case is built on the adversarial population (tests/adversarial.py) with the hold, the remedy hold, tracking,
details and workflow timeouts on a share of records, and compared with the sequential model (tests/handle_model.py)
through a reference handle driven in call order with host ticks (tests/handle_pair.py), which the model checks after
every tick.  The variant with a finite submit budget, which the model does not have, compares with a second handle
driven in call order.  Blobs are read with tests/checkpoint_format.py and tests/checkpoint_delta_format.py.

  1. Calls queued behind device work (one thread): ticks queued behind a delay kernel on a caller stream
     (am_sweep_tick_device, am_sweep_tick_shard, and with staged posts from a posting thread), then a chain's root, a
     delta and a full checkpoint taken without synchronising; ticks queued right after a delta returns, then the next
     delta; a restore behind a queued tick; am_sweep_restore_delta after a tick of every entry point.  A delta's commit
     of a million changed slots, followed at once by the next delta.
  2. A ticker, a poster, a checkpointer and a querier on one source handle whose checkpoints cover 2.2 M slots: a
     root of about 266 MB takes milliseconds to copy while a tick takes a fraction of one.  Only the first 30 000
     slots hold records: a blob's size, which sets the copy's length, is the range's either way, and the model's tick
     over 2.2 M records (about 0.3 s on the host) would make the replay of every tick too slow.  The ticks and posts
     are replayed on the model in their recorded order; every blob is one of two model states; the deltas carry a
     standby that then goes on.
  3. A restore into a handle that another thread ticks at one second.

The stream cases need a GPU; the thread cases also run on the emulated library at a small size
(tests/test_checkpoint_threads_emulator.py)."""
import ctypes
import os
import threading
import time
import zlib

import numpy as np
import pytest

import change_details_oracle
import checkpoint_delta_format as dfmt
import checkpoint_format as fmt
from adversarial import ZoneMap
from handle_pair import DevOut, Pair
from test_checkpoint_gpu import T_PARIS, _fresh, _records, _same_answers

pytestmark = pytest.mark.gpu

EMULATED = "emu" in os.path.basename(os.environ.get("AMSWEEP_LIB", ""))
needs_streams = pytest.mark.skipif(EMULATED, reason="the emulated library completes every call before it returns")

GATE_S = 0.2  # the delay kernel that holds a caller stream
K = 5         # ticks queued behind it
SEED = 7
SWITCHES = dict(hold=True, remedy=True, track=True, details=True)


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def _gate(torch, stream):
    """a delay kernel of about GATE_S on `stream` (it ends by itself); returns an event recorded behind it"""
    done = torch.cuda.Event()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(GATE_S * 2.0e9))  # clock cycles; the H100 runs its SMs at up to 1.98 GHz
        done.record(stream)
    return done


def _busy(am, fn, *a, **kw):
    """fn(*a, **kw), retried while it returns AM_E_BUSY; (result, retries)"""
    retries = 0
    while True:
        try:
            return fn(*a, **kw), retries
        except am.AmError as e:
            if e.code != am.AM_E_BUSY:
                raise
            retries += 1
            time.sleep(0)


def _switch_on(s, budget):
    s.set_seed(SEED)
    s.set_hold_in_flight(True)
    s.set_hold_remedy(True)
    s.set_track_changes(True)
    s.set_change_details(True)
    if budget:
        s.set_submit_budget(budget)


class Twin:
    """the source handle under test and its reference, driven by the same calls: a Pair (a handle and the model,
    compared after every tick), or with a submit budget a second handle.  The reference ticks on the host, in call
    order, and its full checkpoints are the expected blobs."""

    def __init__(self, am, zmap, n, budget=None):
        self.am, self.n, self.budget = am, n, budget
        self.src = am.Sweep(capacity=n)
        _switch_on(self.src, budget)
        if budget:
            self.p, self.ref = None, am.Sweep(capacity=n)
            _switch_on(self.ref, budget)
        else:
            self.p = Pair(am, zmap, n, seed=SEED, every_slot=False, **SWITCHES)
            self.ref = self.p.s

    def close(self):
        self.src.close()
        (self.p or self.ref).close()

    def upsert(self, sl, recs, src=True):
        if src:
            self.src.upsert(sl, recs)
        (self.p or self.ref).upsert(sl, recs)

    def post(self, sl, ph, rp, src=True):
        if src:
            self.src.post_result(sl, ph, rp)
        if self.p:
            self.p.post(sl, ph, rp)
        else:
            self.ref.post_result(sl, ph, rp)

    def tick(self, T, mode=0):
        """the reference's tick: (idx, act, stats)"""
        return tuple(self.p.tick(T, mode)[:3]) if self.p else self.ref.tick(T, mode)

    def full(self, first=0, n=None):
        return self.ref.checkpoint(first, self.n - first if n is None else n)

    def check_model(self, blob):
        """the blob's columns against the model's: flags everywhere, the others on live slots"""
        if not self.p:
            return
        r, m = fmt.read(blob), self.p.m
        live = m.live(np.arange(self.n))
        for name in self.am.COLUMN_NAMES:
            keep = live | (name == "flags")
            np.testing.assert_array_equal(r[name][keep], m.cols()[name][keep], err_msg=name)


def _posts(rng, hwm, k):
    sl = rng.choice(hwm, k).astype(np.uint64)
    return sl, rng.integers(0, 3, k).astype(np.uint8), rng.integers(0, 3, k).astype(np.uint8)


def _issue(s, dev, T, stream):
    s.tick_device(T, 0, dev.ptr[0], dev.ptr[1], dev.n, dev.ptr[2], dev.ptr[3], stream=stream)


def _fetch(am, s, dev):
    idx, act, cnt, st = [a.cpu().numpy() for a in dev.t]
    k = int(cnt.view(np.uint32)[0])
    stats = dict(zip(am.abi.STAT_FIELDS, [int(v) for v in st.view(np.uint64)]))
    return idx.view(np.uint32)[:k].astype(np.uint64) + np.uint64(s.shard_base), act[:k].astype(np.uint32), stats


# ---- 1. calls queued behind device work -------------------------------------------------------------------------
class Queue:
    """K ticks of the source queued behind a delay kernel on a caller stream, through `entry`; with `poster`, a
    posting thread stages results on the source while they wait (its copies still in flight when the next call
    comes).  settle() synchronises, then runs the same ticks and posts on the reference and compares the lists."""

    def __init__(self, torch, am, tw, entry, streams, rng):
        self.torch, self.am, self.tw, self.entry, self.rng = torch, am, tw, entry, rng
        self.stream = streams[1] if entry == "tick_shard" else streams[0]
        self.outs = [DevOut(am, tw.n) for _ in range(K)]

    def issue(self, T0, gate=True):
        s, tw = self.tw.src, self.tw
        if gate:
            self.done = _gate(self.torch, self.stream)
        self.Ts = [T0 + k for k in range(K)]
        for T, dev in zip(self.Ts, self.outs):
            if self.entry == "tick_shard":
                s.tick_shard(T, stream=self.stream.cuda_stream)
            else:
                _issue(s, dev, T, self.stream.cuda_stream)
        self.posts = []
        if self.entry == "poster":
            self.posts = [_posts(self.rng, tw.ref.size, 60) for _ in range(3)]
            t = threading.Thread(target=lambda: [s.post_result(*p) for p in self.posts])
            t.start()
            t.join()
        self.queued = gate and not self.done.query()
        return self.Ts[-1]

    def settle(self):
        self.torch.cuda.synchronize()
        for T, dev in zip(self.Ts, self.outs):
            want = self.tw.tick(T)
            if self.entry != "tick_shard":
                idx, act, st = _fetch(self.am, self.tw.src, dev)
                assert st == want[2], (T, {k: (st[k], want[2][k]) for k in st if st[k] != want[2][k]})
                np.testing.assert_array_equal(idx, want[0], err_msg=f"{T}: idx")
                np.testing.assert_array_equal(act, want[1], err_msg=f"{T}: act")
        for p in self.posts:
            self.tw.post(*p, src=False)


def _stage(tw, rng, zmap, T):
    """a few calls on both handles, staged before the next queued ticks"""
    tw.post(*_posts(rng, tw.ref.size, 40))
    tw.upsert(rng.choice(tw.n, 5).astype(np.uint64), _records(tw.am, zmap, rng, 5, T, True))


def _check_delta(am, delta, k, prev_full, full):
    """the delta's slots are the numpy diff of the reference's full blobs at the two links, and the reader's apply of
    the delta to the previous one gives the new one"""
    d, a, b = dfmt.read(delta), dfmt.read_full(prev_full), dfmt.read_full(full)
    assert d["checksum_ok"] and d["n_changed"] == k == len(d["offsets"])
    np.testing.assert_array_equal(d["offsets"], dfmt.diff(a, b))
    got = dfmt.apply(a, d)
    for name, *_ in dfmt.sections(0, b["switches"])[0]:
        np.testing.assert_array_equal(got[name], b[name], err_msg=name)
    assert got["prev_tick"] == b["prev_tick"] and got["swept_end"] == b["swept_end"]


@needs_streams
@pytest.mark.parametrize("entry,budget", [("tick_device", None), ("tick_shard", None), ("poster", None),
                                          ("tick_device", 3)], ids=["tick_device", "tick_shard", "poster", "budget"])
def test_links_behind_queued_ticks(am, zmap, entry, budget):
    """a root, a delta and a full checkpoint, each taken while K ticks wait behind a delay kernel, must each be the
    state after all K; then a delta, ticks queued on the caller stream as soon as it returns, and the next delta"""
    import torch
    rng = np.random.default_rng(zlib.crc32(f"queued {entry} {budget}".encode()))
    n, T = 3000, T_PARIS
    tw = Twin(am, zmap, n, budget)
    sb = None
    try:
        tw.upsert(np.arange(n - 37, dtype=np.uint64), _records(am, zmap, rng, n - 37, T, True))
        tw.src.tick(T)  # (the kernels are loaded before the first gate)
        tw.tick(T)
        q = Queue(torch, am, tw, entry, (torch.cuda.Stream(), torch.cuda.Stream()), rng)
        queued = []

        # the chain's root
        last = q.issue(T + 1)
        root = tw.src.checkpoint_chain(0, n)
        queued.append(q.queued)
        q.settle()
        assert am.checkpoint_info(root)["prev_tick"] == last
        full = tw.full()
        assert root == full, "root: not the state after the queued ticks"
        tw.check_model(root)
        sb = _fresh(am, n, 0, am.checkpoint_info(root))
        if budget:
            sb.set_submit_budget(budget)
        sb.restore(root)
        _same_answers(am, tw.ref, sb, n, last, "standby from the root")

        # a delta
        _stage(tw, rng, zmap, T)
        last = q.issue(last + 1)
        delta, k = tw.src.checkpoint_delta()
        queued.append(q.queued)
        q.settle()
        assert am.checkpoint_delta_info(delta)["prev_tick"] == last
        prev, full = full, tw.full()
        _check_delta(am, delta, k, prev, full)
        sb.restore_delta(delta)
        assert sb.checkpoint(0, n) == full, "delta: standby differs"

        # a full checkpoint (the chain goes on from the delta's link)
        _stage(tw, rng, zmap, T)
        last = q.issue(last + 1)
        blob = tw.src.checkpoint(0, n)
        queued.append(q.queued)
        q.settle()
        assert blob == tw.full(), "full checkpoint: not the state after the queued ticks"
        tw.check_model(blob)

        # ticks queued (not gated) right after a delta returns, while its commit may still be on the checkpoint
        # stream, then the next delta
        _stage(tw, rng, zmap, T)
        delta, k = tw.src.checkpoint_delta()
        last = q.issue(last + 1, gate=False)
        delta2, k2 = tw.src.checkpoint_delta()
        mid = tw.full()  # (the reference has the staged calls, not yet the ticks)
        q.settle()
        for d, c, a, b in ((delta, k, full, mid), (delta2, k2, mid, tw.full())):
            _check_delta(am, d, c, a, b)
            sb.restore_delta(d)
            assert sb.checkpoint(0, n) == b, f"delta {am.checkpoint_delta_info(d)['seq']}: standby differs"
        assert k2 > 0 and am.checkpoint_delta_info(delta2)["seq"] == 3
        assert all(queued), ("a call returned after its queued ticks had run: nothing was tested", queued)

        # the standby goes on tick for tick
        for t in range(last + 1, last + 4):
            want, got, mine = tw.tick(t), tw.src.tick(t), sb.tick(t)
            for g in (got, mine):
                assert g[2] == want[2] and np.array_equal(g[0], want[0]) and np.array_equal(g[1], want[1]), t
    finally:
        tw.close()
        if sb:
            sb.close()


@needs_streams
def test_next_delta_straight_after_a_large_commit(am):
    """a delta in which every one of 2^20 slots changed, whose commit writes about 100 MB into the base image on the
    checkpoint stream; the next delta is taken straight after it returns, with nothing queued before its diff, and the
    one after that behind a tick queued on a caller stream.  Nothing changes between them but P, so both must carry
    no slot: a diff that read a base image the commit had not finished would list the slots it had not reached.  A
    standby that applies the three links equals the reference."""
    import torch
    n, T = 1 << 20, T_PARIS
    rc, r = am.classify(repeat_after_sec=86400, finished_at=T - 10)
    assert rc == 0
    recs = np.repeat(r, n)
    src, ref, sb = am.Sweep(capacity=n), am.Sweep(capacity=n), None
    A = torch.cuda.Stream()
    dev = DevOut(am, n)
    try:
        for s in (src, ref):
            s.upsert(np.arange(n, dtype=np.uint64), recs)
            s.tick(T)
        root = src.checkpoint_chain(0, n)
        assert root == ref.checkpoint(0, n)
        sb = am.Sweep(capacity=n)
        sb.restore(root)
        need, m = ctypes.c_uint64(0), ctypes.c_uint64(0)
        bufs = [np.ones(len(root) + 4 * n + 4096, np.uint8) for _ in range(3)]  # (faulted in; room for the offsets)

        def delta(buf):
            assert src._lib.am_sweep_checkpoint_delta(src._h, buf.ctypes.data, len(buf), ctypes.byref(need),
                                                      ctypes.byref(m)) == 0
            return need.value, m.value

        prev = root
        for k in range(3):
            recs["finished_at"] = T - 10 + k + 1 + (np.arange(n) % 3)
            for s in (src, ref):
                s.upsert(np.arange(n, dtype=np.uint64), recs)
            links = [delta(bufs[0]), delta(bufs[1])]
            _issue(src, dev, T + 1 + k, A.cuda_stream)
            links.append(delta(bufs[2]))
            torch.cuda.synchronize()
            mid = ref.checkpoint(0, n)
            ref.tick(T + 1 + k)
            full = ref.checkpoint(0, n)
            for (nbytes, c), buf, a, b in zip(links, bufs, (prev, mid, mid), (mid, mid, full)):
                d = buf[:nbytes].tobytes()
                _check_delta(am, d, c, a, b)
                sb.restore_delta(d)
            assert [c for _, c in links] == [n, 0, 0], (k, links)
            assert sb.checkpoint(0, n) == full, k
            prev = full
    finally:
        for s in (src, ref, sb):
            if s:
                s.close()


@needs_streams
def test_restore_behind_a_queued_tick(am, zmap):
    """a restore issued while the standby's tick waits behind a delay kernel on a caller stream: the scatter lands
    after the tick.  The blob carries results posted after the source's tick at the same second, so a tick after the
    scatter would apply them."""
    import torch
    rng = np.random.default_rng(31)
    n, T = 3000, T_PARIS
    tw = Twin(am, zmap, n)
    sb = None
    try:
        tw.upsert(np.arange(n - 37, dtype=np.uint64), _records(am, zmap, rng, n - 37, T, True))
        tw.tick(T)
        root = tw.full()
        sb = _fresh(am, n, 0, am.checkpoint_info(root))
        sb.restore(root)
        calls = _posts(rng, n - 37, 80)  # (on the reference and the standby alike)
        tw.post(*calls, src=False)
        sb.post_result(*calls)
        want = tw.tick(T + 1)
        sl = rng.choice(n // 2, 150).astype(np.uint64)
        tw.post(sl, rng.integers(1, 3, 150).astype(np.uint8), rng.integers(0, 3, 150).astype(np.uint8), src=False)
        blob = tw.full(0, n // 2)
        assert am.checkpoint_info(blob)["prev_tick"] == T + 1
        A = torch.cuda.Stream()
        dev = DevOut(am, n)
        done = _gate(torch, A)
        _issue(sb, dev, T + 1, A.cuda_stream)
        queued = not done.query()
        sb.restore(blob)
        torch.cuda.synchronize()
        idx, act, st = _fetch(am, sb, dev)
        assert st == want[2] and np.array_equal(idx, want[0]) and np.array_equal(act, want[1])
        assert sb.checkpoint(0, n) == tw.full(), "the restore's scatter did not land after the queued tick"
        assert queued
        for t in range(T + 2, T + 5):
            want, got = tw.tick(t), sb.tick(t)
            assert got[2] == want[2] and np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), t
    finally:
        tw.close()
        if sb:
            sb.close()


def test_blob_padding_is_zero(am, zmap):
    """two handles in one state give equal blobs, though one of them staged a blob of another layout before: the
    bytes between a section's last element and its 8-B boundary are zero, not what the earlier blob left in the
    staging area (the restore into a ticking handle below first showed it)"""
    rng = np.random.default_rng(61)
    n, T = 1501, T_PARIS
    recs = _records(am, zmap, rng, n, T, True)
    hs = [am.Sweep(capacity=n) for _ in range(2)]
    try:
        for s in hs:
            _switch_on(s, None)
            s.upsert(np.arange(n, dtype=np.uint64), recs)
            s.tick(T)
        hs[0].checkpoint(3, 700)
        hs[0].checkpoint_chain(1, 1100)
        s0 = hs[0].checkpoint_delta()[0]
        hs[1].checkpoint_chain(1, 1100)
        s1 = hs[1].checkpoint_delta()[0]
        a, b = hs[0].checkpoint(0, n), hs[1].checkpoint(0, n)
        raw = np.frombuffer(a, np.uint8)
        for name, dt, off, nbytes in fmt.sections(n, fmt.read(a)["switches"])[0]:
            assert not raw[off + nbytes:off + (nbytes + 7) // 8 * 8].any(), name
        assert a == b and s0 == s1
        hs[0].post_result(*_posts(rng, n, 333))
        hs[0].checkpoint(5, 3)
        d0 = hs[0].checkpoint_delta()[0]
        r = dfmt.read(d0)
        m = r["n_changed"]
        raw = np.frombuffer(d0, np.uint8)
        for name, dt, off, nbytes in dfmt.sections(m, r["switches"], dfmt.start_of(m))[0]:
            assert not raw[off + nbytes:off + (nbytes + 7) // 8 * 8].any(), name
        assert m % 8  # (sections of u1 and u4 elements end off an 8-B boundary)
    finally:
        for s in hs:
            s.close()


ENTRIES = ["tick", "tick_view", "tick_device", "tick_shard", "run_ticks", "run_ticks_blocked", "simulate"]


def _one_tick(am, s, entry, T):
    if entry == "tick":
        s.tick(T)
    elif entry == "tick_view":
        s.tick_view(T)
    elif entry == "tick_device":
        DevOut(am, s.capacity).tick(am, s, T, 0)
    elif entry == "tick_shard":
        s.tick_shard(T)
    elif entry == "run_ticks":
        s.run_ticks(T, 1)
    elif entry == "run_ticks_blocked":
        s.run_ticks(T, 1, am.SWEEP_BLOCKED)
    else:
        s.simulate(T, 1)


@pytest.mark.parametrize("entry", ENTRIES)
def test_restore_delta_refused_after_a_tick(am, zmap, entry):
    """a standby that ticked once since it applied a delta's parent, through any entry point, refuses the delta with
    AM_E_INVAL and is left as it was; one that did not tick applies it.  (Its P is the delta's after the tick: only the
    tick refuses it.)  am_sweep_run_ticks refuses the hold, so its chain has the hold off."""
    rng = np.random.default_rng(zlib.crc32(entry.encode()))
    n, T = 600, T_PARIS
    hold = not entry.startswith("run_ticks")
    src = am.Sweep(capacity=n)
    stand = []
    try:
        if hold:
            _switch_on(src, None)
        else:
            src.set_track_changes(True)
        src.upsert(np.arange(n, dtype=np.uint64), _records(am, zmap, rng, n, T, hold))
        src.tick(T)
        root = src.checkpoint_chain(0, n)
        src.post_result(*_posts(rng, n, 80))
        src.tick(T + 1)
        delta, k = src.checkpoint_delta()
        assert k > 0
        for _ in range(2):
            stand.append(_fresh(am, n, 0, am.checkpoint_info(root)))
            stand[-1].restore(root)
        ok, sb = stand
        ok.restore_delta(delta)
        assert ok.checkpoint(0, n) == src.checkpoint(0, n)
        _one_tick(am, sb, entry, T + 1)
        before = sb.checkpoint(0, n)
        with pytest.raises(am.AmError) as e:
            sb.restore_delta(delta)
        assert e.value.code == am.AM_E_INVAL, (entry, e.value.code)
        assert sb.checkpoint(0, n) == before, entry
    finally:
        src.close()
        for s in stand:
            s.close()


# ---- 2. a ticker, a poster, a checkpointer and a querier on one source handle -----------------------------------
def _sizes():
    """(slots of the checkpointed range, records in its first slots, ticker's pause in seconds)"""
    return (4096, 1500, 0.0) if EMULATED else (2_200_000, 30_000, 0.002)


class Threads:
    """threads of one case: the first exception of any of them sets `abort`, which every thread's loop checks, and is
    raised by join().  alive() is true while one still runs: its handles must then stay open."""

    def __init__(self):
        self.ts, self.errors, self.abort = [], [], threading.Event()

    def start(self, fn):
        def run():
            try:
                fn()
            except BaseException as e:  # noqa: B036 (re-raised in the main thread)
                self.errors.append(e)
                self.abort.set()
        t = threading.Thread(target=run)
        t.start()
        self.ts.append(t)

    def alive(self):
        return any(t.is_alive() for t in self.ts)

    def join(self):
        for t in self.ts:
            t.join(600)
        assert not self.alive(), "a thread did not finish"
        if self.errors:
            raise self.errors[0]


def _acquire(sem, abort):
    """sem.acquire(), given up (False) once `abort` is set"""
    while not sem.acquire(timeout=0.05):
        if abort.is_set():
            return False
    return True


def _raw_checkpoint(am, s, kind, buf, n):
    """one checkpoint call straight into `buf`: (blob, n_changed or None, start, end, busy retries)"""
    need, m = ctypes.c_uint64(0), ctypes.c_uint64(0)
    retries = 0
    while True:
        t0 = time.perf_counter()
        if kind == "delta":
            rc = s._lib.am_sweep_checkpoint_delta(s._h, buf.ctypes.data, len(buf), ctypes.byref(need), ctypes.byref(m))
        else:
            fn = s._lib.am_sweep_checkpoint_chain if kind == "root" else s._lib.am_sweep_checkpoint
            rc = fn(s._h, 0, n, buf.ctypes.data, len(buf), ctypes.byref(need))
        t1 = time.perf_counter()
        if rc != am.AM_E_BUSY:
            break
        retries += 1
    assert rc == 0, (kind, rc)
    return buf[:need.value].tobytes(), (m.value if kind == "delta" else None), t0, t1, retries


def test_ticker_poster_checkpointer_querier(am, zmap):
    N, S, pause = _sizes()
    rng = np.random.default_rng(41)
    T0 = T_PARIS
    recs = _records(am, zmap, rng, S, T0, True)
    posts = [(rng.choice(S, 50).astype(np.uint64), rng.integers(1, 3, 50).astype(np.uint8),
              rng.integers(0, 3, 50).astype(np.uint8)) for _ in range(1000)]
    src = am.Sweep(capacity=N)
    sb = p = None
    th = Threads()
    try:
        _switch_on(src, None)
        src.upsert(np.arange(S, dtype=np.uint64), recs)
        src.tick(T0)
        need = ctypes.c_uint64(0)
        assert src._lib.am_sweep_checkpoint(src._h, 0, N, None, 0, ctypes.byref(need)) == am.AM_E_NOSPACE
        buf = np.ones(need.value, np.uint8)  # (faulted in before the calls are timed)

        ticks, blobs, busy, done_posts = [], [], {"tick": 0, "checkpoint": 0, "query": 0, "queries": 0}, []
        can_tick, can_post = threading.Semaphore(1), threading.Semaphore(0)
        ck_done, tick_stop = threading.Event(), threading.Event()

        def ticker():
            try:
                tick_loop()
            finally:
                tick_stop.set()
                can_post.release()  # (the poster ends once it has posted after the last tick)
                can_post.release()

        def tick_loop():
            k = 0
            while k < len(posts) - 4 and not (ck_done.is_set() and k >= 3):
                if not _acquire(can_tick, th.abort):
                    return
                T = T0 + 1 + k
                t0 = time.perf_counter()
                (idx, act, st), r = _busy(am, src.tick, T)
                t1 = time.perf_counter()
                (chg, cols), r2 = _busy(am, src.last_changes)
                (didx, det), r3 = _busy(am, src.last_change_details)
                busy["tick"] += r + r2 + r3
                ticks.append(dict(T=T, idx=idx.copy(), act=act.copy(), stats=st, chg=chg, cols=cols, didx=didx,
                                  det=det, t1=t1, t0=t0))
                k += 1
                can_post.release()
                time.sleep(pause)

        def poster():  # exactly one post_result call after every tick
            while True:
                if not _acquire(can_post, th.abort) or len(done_posts) == len(ticks):
                    return
                _busy(am, src.post_result, *posts[len(done_posts)])
                done_posts.append(len(ticks) - 1)
                can_tick.release()

        def checkpointer():
            try:
                blobs.append(("root",) + _raw_checkpoint(am, src, "root", buf, N))
                for j in range(7):
                    if th.abort.is_set():
                        return
                    time.sleep(0.005)
                    blobs.append(("full" if j % 3 == 2 else "delta",) + _raw_checkpoint(
                        am, src, "full" if j % 3 == 2 else "delta", buf, N))
            finally:
                ck_done.set()

        def querier():
            u = np.arange(64, dtype=np.uint64)
            calls = [lambda: src.in_flight(0, 64), lambda: src.remedy_in_flight(idx=u), lambda: src.deferred(0, 64),
                     lambda: src.next_due(T0), lambda: src.repeat_after_sec(T0, 0, 64),
                     lambda: src.last_changes(cap=16)]
            while not tick_stop.is_set() and not th.abort.is_set():
                for c in calls:
                    try:
                        c()
                        busy["queries"] += 1
                    except am.AmError as e:
                        assert e.code == am.AM_E_BUSY, e
                        busy["query"] += 1

        t_start = time.perf_counter()
        for fn in (ticker, poster, checkpointer, querier):
            th.start(fn)
        th.join()
        wall = time.perf_counter() - t_start
        assert tick_stop.is_set() and done_posts == list(range(len(ticks)))
        blobs.append(("delta",) + _raw_checkpoint(am, src, "delta", buf, N))  # (the standby catches up)
        del buf

        # the overlap: ticks that finished while a checkpoint of more than 256 MB was being taken
        calls, over = [], []
        for kind, blob, _, t0, t1, _ in blobs:
            calls.append((kind, len(blob), round((t1 - t0) * 1e3, 2), sum(t0 < t["t1"] < t1 for t in ticks)))
            if len(blob) > 256_000_000:
                over.append(calls[-1])
        print(f"threads: wall {wall:.3f} s, {len(ticks)} ticks, {len(blobs)} blobs, busy retries {busy}, "
              f"median tick {1e3 * float(np.median([t['t1'] - t['t0'] for t in ticks])):.3f} ms, "
              f"checkpoint calls (kind, bytes, ms, ticks that finished during the call) {calls}")
        if not EMULATED:
            assert over and max(o[3] for o in over) >= 1, over

        # the replay, in the recorded order
        p = Pair(am, zmap, N, seed=SEED, every_slot=False, **SWITCHES)
        p.upsert(np.arange(S, dtype=np.uint64), recs)
        p.tick(T0)
        at = {}
        for b in blobs:
            P = (am.checkpoint_info if b[0] != "delta" else am.checkpoint_delta_info)(b[1])["prev_tick"]
            at.setdefault(P - T0 - 1, []).append(b)
        matched = []
        for k in range(-1, len(ticks)):
            if k >= 0:
                t, want = ticks[k], p.tick(ticks[k]["T"])
                assert t["stats"] == want.stats, k
                np.testing.assert_array_equal(t["idx"], want.idx, err_msg=f"tick {k}: idx")
                np.testing.assert_array_equal(t["act"], want.act, err_msg=f"tick {k}: act")
                np.testing.assert_array_equal(t["chg"], p.m.changes(), err_msg=f"tick {k}: changes")
                loc = t["chg"].astype(np.int64)
                for name, a in t["cols"].items():
                    np.testing.assert_array_equal(a, p.m.cols()[name][loc], err_msg=f"tick {k}: {name}")
                np.testing.assert_array_equal(t["didx"], p.m.changes(), err_msg=f"tick {k}: details")
                for name in change_details_oracle.DETAIL.names:
                    np.testing.assert_array_equal(t["det"][name], p.m.details()[name], err_msg=f"tick {k}: {name}")
            if k not in at:
                if k >= 0:
                    p.post(*posts[k])
                continue
            cands = [p.s.checkpoint(0, N)]
            if k >= 0:
                p.post(*posts[k])
                cands.append(p.s.checkpoint(0, N))
                assert cands[0] != cands[1]
            for kind, blob, *_ in at[k]:
                if kind == "root":
                    sb = _fresh(am, N, 0, am.checkpoint_info(blob))
                    sb.set_seed(SEED)
                    sb.restore(blob)
                    got = blob
                elif kind == "full":
                    got = blob
                else:
                    sb.restore_delta(blob)
                    got = sb.checkpoint(0, N)
                hits = [j for j, c in enumerate(cands) if got == c]
                assert len(hits) == 1, (kind, k, hits)
                matched.append((kind, k, ("after the tick", "after the tick and its post")[hits[0]]))
            del cands
        print("blobs matched:", matched)
        assert matched[-1][2] == "after the tick and its post"
        # the standby goes on in the source's place, tick for tick against the model
        p.s.close()
        p.s, sb = sb, None
        for j in range(3):  # (posts[len(ticks)] on are the ones no tick was followed by)
            p.post(*posts[len(ticks) + j])
            p.tick(ticks[-1]["T"] + 1 + j)
    finally:
        if not th.alive():  # (a thread that still calls into the source keeps it open)
            src.close()
        for h in (sb, p):
            if h:
                h.close()


# ---- 3. a restore into a handle that another thread ticks --------------------------------------------------------
def test_restore_into_a_ticking_handle(am, zmap):
    """one thread ticks a handle again and again at the second T of its previous tick (P stays T); another restores
    a blob with P = T over the upper half of its slots, retrying AM_E_BUSY.  The blob carries results posted after
    the tick, so the first tick after the restore applies them: the lists show where it landed, and the handle then
    equals the model with the restore at that point."""
    rng = np.random.default_rng(51)
    n = 1500 if EMULATED else 20_000
    T = T_PARIS
    recs = _records(am, zmap, rng, n, T, True)
    h = am.Sweep(capacity=n)
    q = Pair(am, zmap, n, seed=SEED, every_slot=False, **SWITCHES)
    th = Threads()
    try:
        _switch_on(h, None)
        h.upsert(np.arange(n, dtype=np.uint64), recs)
        h.tick(T)
        q.upsert(np.arange(n, dtype=np.uint64), recs)
        q.tick(T)
        steady = q.tick(T)  # (a tick at the same second again changes nothing)
        assert not any(steady.stats[k] for k in ("n_result_ok", "n_result_fail"))
        sl = (n // 2 + rng.choice(n - n // 2, 300)).astype(np.uint64)
        q.post(sl, rng.integers(1, 3, 300).astype(np.uint8), rng.integers(0, 3, 300).astype(np.uint8))
        blob = q.s.checkpoint(n // 2, n - n // 2)
        assert am.checkpoint_info(blob)["prev_tick"] == T

        got, restored, retries = [], threading.Event(), {}

        def ticker():
            after = 0
            while len(got) < 2000 and after < 3 and not th.abort.is_set():
                r = _busy(am, h.tick, T)[0]
                got.append((r[0].copy(), r[1].copy(), r[2]))
                after += restored.is_set()

        def restorer():
            while len(got) < 3:
                if th.abort.is_set():
                    return
                time.sleep(0.0005)
            retries["restore"] = _busy(am, h.restore, blob)[1]
            restored.set()

        th.start(ticker)
        th.start(restorer)
        th.join()
        assert restored.is_set()
        same = [r[2] == steady.stats and np.array_equal(r[0], steady.idx) for r in got]
        j = same.index(False)
        assert all(same[:j]) and j >= 3, same
        print(f"restore landed after tick {j} of {len(got)}, {retries['restore']} AM_E_BUSY retries")
        for r in got[j:]:
            want = q.tick(T)
            assert r[2] == want.stats and np.array_equal(r[0], want.idx) and np.array_equal(r[1], want.act)
        assert h.checkpoint(0, n) == q.s.checkpoint(0, n)
    finally:
        if not th.alive():
            h.close()
        q.close()
