"""The oracle of a tick with the hold in flight and workflow timeouts (am_record_t.wf_timeout): hold_oracle's tick,
around which the deadlines are kept.  It shares nothing with the device's segment bounds.

Per slot: `wf`, the workflow timeout W of the slot's latest upsert (0 after a load), and `deadline`, the running
workflow's deadline D or NO_DEADLINE.  A tick at T:
  * before it, every slot with D <= T that is held (hold_oracle.held) and live (kinds 1..5, not a tombstone) is posted
    Failed, as am_sweep_post_result(slot, AM_PHASE_FAILED, AM_PHASE_NONE) would be — the C oracle's pending bits, and
    hold_oracle.post for since; then every D <= T is dropped;
  * then hold_oracle.sweep;
  * after it, every slot the tick submitted gets D = T + W when W > 0, else none.
A remove, a load and turning the hold on drop D (tests/handle_model.py keeps all of it for one handle, in call order)."""
import numpy as np

import hold_oracle

NO_DEADLINE = (1 << 63) - 1
KIND_MASK = 0x7
F_PENDING_OK, F_PENDING_FAIL = 1 << 4, 1 << 5
F_TOMBSTONE = 1 << 8
ACT_SUBMIT_HC = 0x01
PHASE_FAILED = 2


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
