"""The oracle of a tick with the hold in flight on (am_sweep_set_hold_in_flight): the C oracle's tick (orc_sweep, or
the window oracle's catch-up tick) around which the holds are kept.

`since[i]` is the second of the tick that submitted slot i's running health-check workflow, or NOT_IN_FLIGHT.  A
workflow phase posted for the slot, a remove and a load clear it (`post`, `clear`) — a posted phase whatever follows
it before the tick (an upsert that supersedes the result, a tick second not later than since).  A record is held when
since is set, since >= finishedAt and no workflow phase (Succeeded / Failed) is pending.  For the one call:
  * held records whose kind can be due (INTERVAL, CRON_EVERY, CRON_SPEC) are rewritten so that they are not: an
    interval check with its timer armed, finishedAt = T and RepeatAfterSec = INT32_MAX (zone bits cleared).  Held
    STOPPED and PARSE_ERROR records are left alone, so their actions still come out;
  * kind, zone, interval, masks, the timer bit and finishedAt are restored afterwards.  orc_sweep writes none of them
    for such a record: it has no workflow phase pending, so no result re-arms its timer or sets its finishedAt;
  * every returned entry with SUBMIT_HC gets since := T.
It relies on the property the window oracle documents: after the due decision nothing depends on kind or interval.
"""
import numpy as np

import window_oracle

KIND_MASK, KIND_INTERVAL, KIND_CRON_SPEC, KIND_CRON_EVERY = 0x7, 2, 3, 4
F_PENDING_OK, F_PENDING_FAIL = 1 << 4, 1 << 5
F_TOMBSTONE, F_TIMER_ARMED = 1 << 8, 1 << 10
TZ_SHIFT = 24
ACT_SUBMIT_HC = 0x01
I32MAX = (1 << 31) - 1
NOT_IN_FLIGHT = -(1 << 63)
MASKS = ("minute", "hour", "dom", "month", "dow")


def none_in_flight(n):
    return np.full(n, NOT_IN_FLIGHT, dtype=np.int64)


def held(ocols, since):
    """bool[n]: the rule of the sweep (and of am_sweep_in_flight) on the state as it stands"""
    f = ocols["flags"]
    pend = (f & np.uint32(F_PENDING_OK | F_PENDING_FAIL)) != 0
    return (since != NOT_IN_FLIGHT) & (since >= ocols["finished_at"]) & ~pend


def in_flight(ocols, since):
    """what am_sweep_in_flight returns for every slot"""
    return np.where(held(ocols, since), since, np.int64(NOT_IN_FLIGHT))


def sweep(zmap, ocols, since, T, P=None, mode=0, seed=0, shard_base=0):
    """The tick at T with the hold on, IN PLACE on the columns and on `since` (int64[n], local slots).  P: the previous
    tick's second for a catch-up tick (AM_SWEEP_CATCH_UP), else None.  Open loop only (mode bit 0 clear).  Returns
    (global idx, action, stats) like oracle_c.sweep."""
    assert not (mode & 1), "a closed-loop tick is refused while the hold is on"
    f0 = ocols["flags"].copy()
    kind = f0 & np.uint32(KIND_MASK)
    live = (f0 & np.uint32(F_TOMBSTONE)) == 0
    can_be_due = (kind == KIND_INTERVAL) | (kind == KIND_CRON_EVERY) | (kind == KIND_CRON_SPEC)
    h = held(ocols, since) & can_be_due & live
    saved = {k: ocols[k][h].copy() for k in ("flags", "ras", "finished_at") + MASKS}
    keep = np.uint32(~(KIND_MASK | (0xFF << TZ_SHIFT)) & 0xFFFFFFFF)
    ocols["flags"][h] = (f0[h] & keep) | np.uint32(KIND_INTERVAL | F_TIMER_ARMED)
    ocols["ras"][h] = I32MAX
    ocols["finished_at"][h] = T
    try:
        if P is None:
            out = zmap.sweep(ocols, T, mode=mode, seed=seed, shard_base=shard_base)
        else:
            out = window_oracle.sweep_window(zmap, ocols, P, T, mode=mode, seed=seed, shard_base=shard_base)
    finally:
        for k, v in saved.items():
            if k != "flags":
                ocols[k][h] = v
        # (a remedy phase applied by the call cleared its bits: only kind, zone and the timer bit go back)
        back = np.uint32(KIND_MASK | (0xFF << TZ_SHIFT) | F_TIMER_ARMED)
        ocols["flags"][h] = (ocols["flags"][h] & ~back) | (saved["flags"] & back)
    idx, act, _ = out
    sub = (np.asarray(act) & ACT_SUBMIT_HC) != 0
    since[np.asarray(idx, dtype=np.int64)[sub] - int(shard_base)] = T
    return out


def post(since, slots, phase):
    """am_sweep_post_result of `slots` (local) with workflow phases `phase` (0 = none: a remedy phase alone)"""
    slots = np.asarray(slots, dtype=np.int64)
    since[slots[np.asarray(phase) != 0]] = NOT_IN_FLIGHT


def clear(since, slots):
    """am_sweep_remove / am_sweep_load_range of `slots` (local)"""
    since[np.asarray(slots, dtype=np.int64)] = NOT_IN_FLIGHT
