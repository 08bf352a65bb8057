"""The oracle of a tick with the hold in flight, workflow timeouts and the remedy hold on (am_sweep_set_hold_remedy):
timeout_oracle's tick, around which the remedy runs are kept.  It shares nothing with the device's encoding (one since
word and one deadline word per slot for both kinds of run): the remedy runs have arrays of their own.

Per slot: `rsince`, the start of the running remedy workflow or NOT_IN_FLIGHT, and `rdeadline`, its deadline or
NO_DEADLINE.  A remedy run is HELD when rsince is set and no workflow phase is pending (hold_oracle's rule with the run in
place of since).  A tick at T:
  1. every slot with rdeadline <= T that is held and live gets a posted remedy "Failed", as
     am_sweep_post_result(slot, AM_PHASE_NONE, AM_PHASE_FAILED) would (the C oracle's pending bits); its run ends; every
     rdeadline <= T is dropped;
  2. held remedy runs are shown to timeout_oracle.sweep as held health-check runs (a since that is always >= finishedAt);
  3. after the call every entry with RUN_REMEDY whose flags before the call had no REMEDY_PENDING starts a run at T: its
     SUBMIT_HC is dropped and n_submit_hc decremented (an open-loop submit writes no column), rsince = T,
     rdeadline = T + W when the slot's W > 0, and the health-check since and deadline are cleared; every entry still
     submitted ends the slot's remedy run (a check has one run in flight).
A posted workflow or remedy phase, a remove, a load and toggling either hold end a remedy run; an upsert does not
(tests/handle_model.py keeps the runs for one handle, in call order)."""
import numpy as np

import hold_oracle
import timeout_oracle

NONE = hold_oracle.NOT_IN_FLIGHT
NO_DEADLINE = timeout_oracle.NO_DEADLINE
F_PENDING_OK, F_PENDING_FAIL = 1 << 4, 1 << 5
F_REMEDY_PENDING, F_REMEDY_OUTCOME_OK = 1 << 6, 1 << 7
ACT_SUBMIT_HC, ACT_RUN_REMEDY = 0x01, 0x02
ALWAYS_HELD = 1 << 62  # a since that is >= every finishedAt a test uses


def held(ocols, rsince):
    """bool[n]: remedy runs the next tick holds"""
    pend = (ocols["flags"] & np.uint32(F_PENDING_OK | F_PENDING_FAIL)) != 0
    return (rsince != NONE) & ~pend


def in_flight(ocols, rsince):
    """what am_sweep_remedy_in_flight returns for every slot"""
    return np.where(held(ocols, rsince), rsince, np.int64(NONE))


def expire(ocols, rsince, rdeadline, T, shard_base=0):
    """step 1, IN PLACE.  Returns (global idx u64, start i64) of the timed-out remedy runs."""
    due = rdeadline <= T
    sl = np.flatnonzero(due & held(ocols, rsince) & timeout_oracle.live(ocols["flags"]))
    out = (sl.astype(np.uint64) + np.uint64(shard_base), rsince[sl].copy())
    f = ocols["flags"]
    f[sl] = (f[sl] & np.uint32(~(F_REMEDY_PENDING | F_REMEDY_OUTCOME_OK) & 0xFFFFFFFF)) | np.uint32(F_REMEDY_PENDING)
    rsince[sl] = NONE
    rdeadline[due] = NO_DEADLINE
    return out


def sweep(zmap, ocols, since, deadline, wf, rsince, rdeadline, T, P=None, shard_base=0):
    """The tick at T, IN PLACE.  Returns (global idx, action, stats, timed_out, remedy_timed_out)."""
    rtimed = expire(ocols, rsince, rdeadline, T, shard_base)
    running = rsince != NONE
    assert (since[running] == NONE).all() and (deadline[running] == NO_DEADLINE).all(), "one run per check"
    shown = np.where(running, np.int64(ALWAYS_HELD), since)
    pre = ocols["flags"].copy()
    idx, act, st, timed = timeout_oracle.sweep(zmap, ocols, shown, deadline, wf, T, P=P, shard_base=shard_base)
    act = np.asarray(act).copy()
    st = dict(st)
    loc = np.asarray(idx, dtype=np.int64) - int(shard_base)
    start = ((act & ACT_RUN_REMEDY) != 0) & ((pre[loc] & np.uint32(F_REMEDY_PENDING)) == 0)
    st["n_submit_hc"] -= int(((act & ACT_SUBMIT_HC) != 0)[start].sum())
    act[start] &= np.uint32(~ACT_SUBMIT_HC & 0xFFFFFFFF)
    sub = loc[(act & ACT_SUBMIT_HC) != 0]
    rsince[sub] = NONE
    rdeadline[sub] = NO_DEADLINE
    sl = loc[start]
    shown[sl] = NONE
    deadline[sl] = NO_DEADLINE
    rsince[sl] = T
    w = wf[sl].astype(np.int64)
    rdeadline[sl] = np.where(w > 0, T + w, NO_DEADLINE)
    since[:] = np.where(shown == ALWAYS_HELD, np.int64(NONE), shown)
    return idx, act, st, timed, rtimed
