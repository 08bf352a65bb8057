"""The oracle of a tick with the hold in flight and workflow timeouts (am_record_t.wf_timeout): hold_oracle's tick,
around which the deadlines are kept.  It shares nothing with the device's segment bounds.

Per slot: `wf`, the workflow timeout W of the slot's latest upsert (0 after a load), and `deadline`, the running
workflow's deadline D or NO_DEADLINE.  A tick at T:
  * before it, every slot with D <= T that is held (hold_oracle.held) and live (kinds 1..5, not a tombstone) is posted
    Failed, as am_sweep_post_result(slot, AM_PHASE_FAILED, AM_PHASE_NONE) would be — the C oracle's pending bits, and
    hold_oracle.post for since; then every D <= T is dropped;
  * then hold_oracle.sweep;
  * after it, every slot the tick submitted gets D = T + W when W > 0, else none.
A remove, a load and turning the hold on drop D.  `State` keeps all of it for one handle, in call order."""
import numpy as np

import hold_oracle
import oracle_c

NO_DEADLINE = (1 << 63) - 1
KIND_MASK = 0x7
F_PENDING_OK, F_PENDING_FAIL = 1 << 4, 1 << 5
F_REMEDY_PENDING, F_REMEDY_OUTCOME_OK = 1 << 6, 1 << 7
F_TOMBSTONE = 1 << 8
ACT_SUBMIT_HC = 0x01
PHASE_SUCCEEDED, PHASE_FAILED = 1, 2
CATCH_UP = 0x8
COLUMN_NAMES = [n for n, _ in oracle_c.COLUMNS]


def no_deadlines(n):
    return np.full(n, NO_DEADLINE, dtype=np.int64)


def live(flags):
    """kinds 1..5 and not a tombstone: the records a tick evaluates"""
    kind = flags & np.uint32(KIND_MASK)
    return (kind >= 1) & (kind <= 5) & ((flags & np.uint32(F_TOMBSTONE)) == 0)


def expire(ocols, since, deadline, T, shard_base=0):
    """The expiry before the tick at T, IN PLACE.  Returns (global idx u64, since i64) of the timed-out runs."""
    due = deadline <= T
    sl = np.flatnonzero(due & hold_oracle.held(ocols, since) & live(ocols["flags"]))
    out = (sl.astype(np.uint64) + np.uint64(shard_base), since[sl].copy())
    f = ocols["flags"]
    f[sl] = (f[sl] & np.uint32(~(F_PENDING_OK | F_PENDING_FAIL) & 0xFFFFFFFF)) | np.uint32(F_PENDING_FAIL)
    hold_oracle.post(since, sl, np.full(len(sl), PHASE_FAILED, dtype=np.uint8))
    deadline[due] = NO_DEADLINE
    return out


def sweep(zmap, ocols, since, deadline, wf, T, P=None, mode=0, seed=0, shard_base=0):
    """The tick at T with the hold on and timeouts, IN PLACE.  Returns (global idx, action, stats, timed_out)."""
    timed = expire(ocols, since, deadline, T, shard_base)
    idx, act, st = hold_oracle.sweep(zmap, ocols, since, T, P=P, mode=mode, seed=seed, shard_base=shard_base)
    loc = np.asarray(idx, dtype=np.int64)[(np.asarray(act) & ACT_SUBMIT_HC) != 0] - int(shard_base)
    w = wf[loc].astype(np.int64)
    deadline[loc] = np.where(w > 0, T + w, NO_DEADLINE)
    return idx, act, st, timed


def first_event(zmap, ocols, since, deadline, wf, T, horizon):
    """the first second of (T, T + horizon] at which a plain tick emits anything, applies a result or times a run out,
    by brute force over copies; None when there is none"""
    c = {k: v.copy() for k, v in ocols.items()}
    s, d = since.copy(), deadline.copy()
    for t in range(T + 1, T + horizon + 1):
        idx, _, st, timed = sweep(zmap, c, s, d, wf, t)
        if len(idx) or len(timed[0]) or st["n_result_ok"] or st["n_result_fail"] or st["n_remedy_ok"] or st["n_remedy_fail"]:
            return t
    return None


class State:
    """the oracle side of one handle with the hold on: columns, since, W and D per slot, and P (the previous tick)"""

    def __init__(self, zmap, cols, shard_base=0):
        self.zmap = zmap
        self.ocols = {k: np.ascontiguousarray(v).copy() for k, v in cols.items()}
        self.n = len(self.ocols["flags"])
        self.since = hold_oracle.none_in_flight(self.n)
        self.deadline = no_deadlines(self.n)
        self.wf = np.zeros(self.n, dtype=np.int32)
        self.shard_base = shard_base
        self.P = None

    def upsert(self, slots, recs):
        for k, i in enumerate(np.asarray(slots, dtype=np.int64)):  # in call order: a later entry of the slot wins
            for name in COLUMN_NAMES:
                self.ocols[name][i] = recs[name][k]
            self.ocols["flags"][i] &= np.uint32(~F_TOMBSTONE & 0xFFFFFFFF)
            self.wf[i] = recs["wf_timeout"][k]

    def remove(self, slots):
        slots = np.asarray(slots, dtype=np.int64)
        self.ocols["flags"][slots] = F_TOMBSTONE
        hold_oracle.clear(self.since, slots)
        self.deadline[slots] = NO_DEADLINE

    def post(self, slots, phase, rphase=None):
        slots = np.asarray(slots, dtype=np.int64)
        phase = np.asarray(phase, dtype=np.uint8)
        hc = np.uint32(F_PENDING_OK | F_PENDING_FAIL)
        rm = np.uint32(F_REMEDY_PENDING | F_REMEDY_OUTCOME_OK)
        for k, i in enumerate(slots):
            f = self.ocols["flags"][i]
            if phase[k]:
                f = (f & ~hc) | np.uint32(F_PENDING_OK if phase[k] == PHASE_SUCCEEDED else F_PENDING_FAIL)
            if rphase is not None and rphase[k]:
                f = (f & ~rm) | (rm if rphase[k] == PHASE_SUCCEEDED else np.uint32(F_REMEDY_PENDING))
            self.ocols["flags"][i] = f
        hold_oracle.post(self.since, slots, phase)

    def load(self, first, cols):
        m = len(cols["flags"])
        for name in COLUMN_NAMES:
            self.ocols[name][first:first + m] = cols[name]
        sl = np.arange(first, first + m)
        hold_oracle.clear(self.since, sl)
        self.wf[first:first + m] = 0
        self.deadline[first:first + m] = NO_DEADLINE

    def hold_on_again(self):
        """am_sweep_set_hold_in_flight off, then on: nothing in flight, no deadline"""
        self.since[:] = hold_oracle.NOT_IN_FLIGHT
        self.deadline[:] = NO_DEADLINE

    def tick(self, T, mode=0):
        P = self.P if (mode & CATCH_UP) and self.P is not None and T > self.P else None
        out = sweep(self.zmap, self.ocols, self.since, self.deadline, self.wf, T, P=P, shard_base=self.shard_base)
        self.P = T
        return out

    def in_flight(self):
        return hold_oracle.in_flight(self.ocols, self.since)

    def next_event(self, T, horizon):
        return first_event(self.zmap, self.ocols, self.since, self.deadline, self.wf, T, horizon)
