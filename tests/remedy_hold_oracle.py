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
A posted workflow or remedy phase, a remove, a load and toggling either hold end a remedy run; an upsert does not.
With the remedy hold off the state is timeout_oracle.State's alone."""
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


def first_event(zmap, ocols, since, deadline, wf, rsince, rdeadline, T, horizon):
    """the first second of (T, T + horizon] at which a plain tick emits anything, applies a result or times a run of
    either kind out, by brute force over copies; None when there is none"""
    c = {k: v.copy() for k, v in ocols.items()}
    s, d, rs, rd = since.copy(), deadline.copy(), rsince.copy(), rdeadline.copy()
    for t in range(T + 1, T + horizon + 1):
        idx, _, st, timed, rtimed = sweep(zmap, c, s, d, wf, rs, rd, t)
        if (len(idx) or len(timed[0]) or len(rtimed[0]) or st["n_result_ok"] or st["n_result_fail"] or st["n_remedy_ok"]
                or st["n_remedy_fail"]):
            return t
    return None


class State(timeout_oracle.State):
    """the oracle side of one handle with the hold on: timeout_oracle.State plus the remedy runs and the switch"""

    def __init__(self, zmap, cols, shard_base=0, remedy=True):
        super().__init__(zmap, cols, shard_base)
        self.rsince = hold_oracle.none_in_flight(self.n)
        self.rdeadline = timeout_oracle.no_deadlines(self.n)
        self.remedy = remedy

    def _end(self, slots):
        self.rsince[slots] = NONE
        self.rdeadline[slots] = NO_DEADLINE

    def remove(self, slots):
        super().remove(slots)
        self._end(np.asarray(slots, dtype=np.int64))

    def post(self, slots, phase, rphase=None):
        super().post(slots, phase, rphase)
        slots = np.asarray(slots, dtype=np.int64)
        ends = np.asarray(phase) != 0
        if rphase is not None:
            ends |= np.asarray(rphase) != 0
        self._end(slots[ends])

    def load(self, first, cols):
        super().load(first, cols)
        self._end(np.arange(first, first + len(cols["flags"])))

    def hold_on_again(self):
        """am_sweep_set_hold_in_flight off, then on: the remedy hold is off as well"""
        super().hold_on_again()
        self._end(slice(None))
        self.remedy = False

    def set_remedy(self, on):
        """am_sweep_set_hold_remedy while the hold is on"""
        if not on:
            self._end(slice(None))
        self.remedy = bool(on)

    def tick(self, T, mode=0):
        """(global idx, action, stats, timed_out, remedy_timed_out)"""
        P = self.P if (mode & timeout_oracle.CATCH_UP) and self.P is not None and T > self.P else None
        if self.remedy:
            out = sweep(self.zmap, self.ocols, self.since, self.deadline, self.wf, self.rsince, self.rdeadline, T, P=P,
                        shard_base=self.shard_base)
        else:
            out = timeout_oracle.sweep(self.zmap, self.ocols, self.since, self.deadline, self.wf, T, P=P,
                                       shard_base=self.shard_base)
            out = out + ((np.zeros(0, dtype=np.uint64), np.zeros(0, dtype=np.int64)),)
        self.P = T
        return out

    def remedy_in_flight(self):
        return in_flight(self.ocols, self.rsince)

    def next_event(self, T, horizon):
        if not self.remedy:
            return super().next_event(T, horizon)
        return first_event(self.zmap, self.ocols, self.since, self.deadline, self.wf, self.rsince, self.rdeadline, T,
                           horizon)
