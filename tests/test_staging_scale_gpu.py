"""Drains that cross the staging arrays' early host-to-device copies (kFlushOps = 32768 ops, kFlushRecs = 8192 upsert
and spec-update records), with the hold, the remedy hold, workflow timeouts, tracking, change details and a finite
submit budget on, against tests/spec_update_model.py through tests/test_spec_update_gpu.py's SpecPair, compared after
every tick.  In every drain a set of slots gets its upsert, which fills a records chunk on its own and so leaves in an
early copy, then a post call of more than one ops chunk, then its spec update, which leaves in a later copy, then a
remove of some of them in a later ops copy than their upserts, and posts after it.  The test follows the host's flush
rules and asserts where each of these went.  One drain is staged from four threads at once on disjoint slot sets, so
that their ranges complete out of order."""
import threading
import zlib

import numpy as np
import pytest

from adversarial import population, zones_usable
from test_spec_update_gpu import NONE, SpecPair, zmap  # noqa: F401 (zmap: the module's fixture)
from timeout_cases import M0

pytestmark = pytest.mark.gpu

FLUSH_OPS, FLUSH_RECS = 32768, 8192  # csrc/sweep.cu kFlushOps, kFlushRecs
OP_BYTES, REC_BYTES = 8, 96  # a staged op, an am_record_t
DAY = 86400
STEPS = [1, 59, 1, 60, 0, 1, -30, 1, 61]
X = 300  # slots per drain whose calls straddle the copies


def _reserve(cap, nbytes):
    """a device twin's bytes after DevBuf::reserve(nbytes) (csrc/sweep.cu)"""
    return cap if nbytes <= cap else nbytes + nbytes // 2 + 4096


class StagingPair(SpecPair):
    """SpecPair that follows what each drain stages and where the host hands it to the copy stream: the flush rules of
    csrc/sweep.cu (flush_staging at the end of an upsert, spec update or remove; at each full chunk inside a post call
    with more of the call behind it, and, ops only, at its end) over the device twins that the previous drain of the
    same staging area left.  Per drain: the ops and records, the calls (call, first op, entries, first record), the
    early copies (kind, lo, hi) and whether threads staged it.  A drain that grows its twins copies everything again:
    none of its early copies count."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.twins = [[0, 0], [0, 0]]  # per staging area: bytes of the device ops and records
        self.area = 0
        self.drains = []
        self._reset()

    def _reset(self):
        self.ops = self.recs = self.fl_ops = self.fl_recs = 0
        self.log, self.copies, self.threaded = [], [], False

    def _flush(self, upto=None, recs=True):
        upto = self.ops if upto is None else upto
        ops_cap, recs_cap = self.twins[self.area]
        if upto - self.fl_ops >= FLUSH_OPS and ops_cap >= upto * OP_BYTES:
            self.copies.append(("ops", self.fl_ops, upto))
            self.fl_ops = upto
        if recs and self.recs - self.fl_recs >= FLUSH_RECS and recs_cap >= self.recs * REC_BYTES:
            self.copies.append(("recs", self.fl_recs, self.recs))
            self.fl_recs = self.recs

    def _note(self, call, k, recs=False):
        self.log.append((call, self.ops, k, self.recs if recs else None))
        self.ops += k
        self.recs += k if recs else 0

    def upsert(self, slots, recs):
        self._note("upsert", len(slots), True)
        super().upsert(slots, recs)
        self._flush()

    def update_spec(self, slots, recs):
        self._note("spec", len(slots), True)
        super().update_spec(slots, recs)
        self._flush()

    def remove(self, slots):
        self._note("remove", len(slots))
        super().remove(slots)
        self._flush()

    def post(self, slots, phase, rphase=None):
        a, k = self.ops, len(slots)
        self._note("post", k)
        super().post(slots, phase, rphase)
        for end in range(a + FLUSH_OPS, a + k, FLUSH_OPS):
            self._flush(end)
        self._flush(recs=False)

    def tick(self, T, mode=0, entry=None):
        tw = self.twins[self.area]
        if tw[0] < self.ops * OP_BYTES or tw[1] < self.recs * REC_BYTES:
            tw[:] = _reserve(tw[0], self.ops * OP_BYTES), _reserve(tw[1], self.recs * REC_BYTES)
            self.copies = []
        self.drains.append((self.ops, self.recs, self.log, self.copies, self.threaded))
        self.area ^= 1
        self._reset()
        return super().tick(T, mode, entry)


def _copy_of(copies, kind, lo, hi):
    """the index of the early copy that holds [lo, hi) of `kind`, len(copies) for the drain's final copy, None when the
    range is split between copies"""
    for j, (c, a, b) in enumerate(copies):
        if c == kind and a <= lo and hi <= b:
            return j
    done = max([b for c, _, b in copies if c == kind], default=0)
    return len(copies) if lo >= done else None


def _crossing(log, copies):
    """True when the upsert's last X records (the straddling slots) leave in one copy and the same slots' spec update in
    a later one, a post call of more than an ops chunk lies between them, and the remove of some of the slots leaves in
    a later ops copy than their upserts"""
    (u, u_op, k, u_rec), (b, _, big, _), (s, _, ks, s_rec), _, (x, x_op, kx, _) = log[:5]
    ur, sr = _copy_of(copies, "recs", u_rec + k - X, u_rec + k), _copy_of(copies, "recs", s_rec + ks - X, s_rec + ks)
    uo, xo = _copy_of(copies, "ops", u_op + k - X, u_op + k), _copy_of(copies, "ops", x_op, x_op + kx)
    return ((u, b, s, x) == ("upsert", "post", "spec", "remove") and big > FLUSH_OPS and None not in (ur, sr, uo, xo)
            and ur < sr and uo < xo)


def test_drains_across_the_flush_chunks(am, zmap):
    n = 20_000
    rng = np.random.default_rng(zlib.crc32(b"staging scale"))
    T = M0 + 5 * DAY + 13 * 3600 - 1
    zones = zmap.ids_of(zones_usable(T - DAY, T + 2 * DAY))
    p = StagingPair(am, zmap, n, hold=True, remedy=True, track=True, details=True, every_slot=False)

    def records(k):
        r = am.columns_to_records(population(rng, k, T, True, zones))
        r["wf_timeout"] = np.where(rng.random(k) < 0.3, 0, rng.integers(1, 200, k))
        return r

    def phases(k):
        return rng.integers(0, 3, k).astype(np.uint8), rng.integers(0, 3, k).astype(np.uint8)

    def busy_first(k):
        """k slots: the ones in flight first (their runs end), then random ones, duplicates included"""
        busy = rng.permutation(np.flatnonzero(p.m.since[:n] != NONE))[:k // 2]
        return np.concatenate([busy, rng.integers(0, n, k - len(busy))])

    try:
        p.set_budget(400)
        p.upsert(np.arange(n), records(n))
        p.tick(T)
        for k, step in enumerate(STEPS):
            if k % 3 == 2:
                p.set_budget([0, 25, 900, 3000][k % 4])
            x = rng.choice(n, X, replace=False)
            filler = rng.integers(0, n, FLUSH_RECS)  # (the upsert alone fills a records chunk, x last)
            p.upsert(np.concatenate([filler, x]), records(len(filler) + len(x)))
            p.post(busy_first(FLUSH_OPS + 4_000), *phases(FLUSH_OPS + 4_000))
            p.update_spec(np.concatenate([rng.integers(0, n, 900), x]), records(1_200))
            p.post(busy_first(FLUSH_OPS - 5_000), *phases(FLUSH_OPS - 5_000))
            p.remove(x[:40])
            p.post(np.concatenate([x, busy_first(500)]), *phases(800))
            if k == 4:
                _threads(p, rng, records, phases)
            T += step
            p.tick(T, entry=["tick", "tick_view", "tick_device", "tick_shard"][k % 4])
        crossed = 0
        for j, (ops, recs, log, copies, threaded) in enumerate(p.drains[1:], 1):
            assert ops > 2 * FLUSH_OPS and recs > FLUSH_RECS, (ops, recs)
            # (the first drain of each staging area, and the second of area 0, size its twins; the threaded drain's
            # ranges complete in no fixed order)
            if j >= 3 and not threaded:
                assert _crossing(log, copies), (j, log[:5], copies)
                crossed += 1
        assert crossed >= 5 and p.drains[5][4] and p.drains[5][0] > 4 * FLUSH_OPS, (crossed, p.drains[5][:2])
        assert p.detailed > 50_000 and p.started > 500, (p.detailed, p.started)
    finally:
        p.close()


def _threads(p, rng, records, phases):
    """four threads, each with its own quarter of the slots: an upsert, a post of more than an ops chunk, a spec update,
    a remove and a post, concurrently with the others; then the model takes each thread's calls in its order"""
    n = p.n
    parts = np.array_split(rng.permutation(n), 4)
    plans = []
    for sl in parts:
        big = rng.choice(sl, FLUSH_OPS + 1_000)
        plans.append([("upsert", sl[:2_500], records(2_500)), ("post", big, *phases(len(big))),
                      ("update_spec", sl[1_000:2_000], records(1_000)), ("remove", sl[:20]),
                      ("post", sl[:3_000], *phases(3_000))])

    def run(plan):
        for call, *args in plan:
            getattr(p.s, "post_result" if call == "post" else call)(*args)

    ts = [threading.Thread(target=run, args=(plan,)) for plan in plans]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    p.threaded = True
    for plan in plans:
        for call, *args in plan:
            getattr(p.m, call)(*args)
            p._note(call, len(args[0]), call in ("upsert", "update_spec"))
