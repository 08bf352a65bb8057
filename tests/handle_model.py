"""One sequential model of a sweep handle, built only from the per-tick oracles: the oracle side of every suite that
drives a handle (the hand-derived cases run on it alone) and of every random call sequence.

State: the sixteen columns of every slot (in the product's zone ids, like adversarial.ZoneMap), the high-water mark of
the swept slots, the previous tick's second P and the seed; the switches hold, remedy hold, tracking and details; per
slot the hold's `since`, the workflow timeout W of the slot's latest upsert (0 after a load), the running workflow's
deadline D, the running remedy run's start and deadline, and the starts the details take at the posts; the last tick's
timed-out lists, changed set and details.

Calls apply in call order (DESIGN §6 item 9):
  * upsert / remove / post / load change the columns at once.  A posted phase replaces its bit group of the pending
    bits the next tick applies (the latest entry of a slot wins), so a later upsert or load of the slot supersedes it.
    A workflow phase, a remove and a load clear since; a remove and a load drop D; a posted workflow or remedy phase, a
    remove and a load end a remedy run, an upsert does not.  With details on, a post first takes in_flight() and
    remedy_in_flight() of its slots for the phases it stages; an upsert, remove or load of a slot drops what was taken.
    A read drains on the handle and changes nothing here.
  * set_hold: turning it on leaves nothing in flight and no deadline; turning it off turns the remedy hold off.
    set_remedy (refused while the hold is off): turning it off ends every remedy run.  set_track: turning it off turns
    details off; turning it on starts an empty changed set.  set_details (refused while tracking is off) drops what
    was taken, and turning it on starts with no details.
  * a tick at T is a catch-up tick over (P, T] when CATCH_UP is set, P is set and T > P.  It sweeps the slots below the
    high-water mark: with the remedy hold remedy_hold_oracle.sweep, with the hold timeout_oracle.sweep (expiry, then
    hold_oracle.sweep), else window_oracle.sweep_window or the plain oracle.  With tracking it lists
    changes_oracle.changed, with details change_details_oracle.details of the listed slots.  It returns
    Tick(idx, act, stats, timed_out, remedy_timed_out); both lists are empty without the hold.
  * run_ticks is the plain oracle's tick at T0 .. T0 + n - 1; it tracks nothing and empties the changed set.
  * a refused call raises Refused(code) and changes nothing: a closed-loop tick with the hold on, a catch-up window
    longer than a day (AM_E_RANGE), run_ticks with the hold or CATCH_UP, set_remedy without the hold, set_details
    without tracking.  P follows DESIGN §6 item 11: every successful tick sets it, one that returns AM_E_NOSPACE
    included; run_ticks sets it to its last second; refusals leave it.
Queries: in_flight / remedy_in_flight (hold_oracle / remedy_hold_oracle, NOT_IN_FLIGHT without their hold);
repeat_after (interval and "@every": the stored interval; a UTC 5-field schedule: the C oracle's
orc_cron_repeat_after_sec; one bound to a named zone: the Python oracle's "first instant whose wall clock matches",
DESIGN §6 item 10; everything else, tombstones included, 0); first_active_tick (the first plain tick that emits, applies
a result or times a run of either kind out, by brute force over copies)."""
import ctypes as C
from collections import namedtuple

import numpy as np

import change_details_oracle
import changes_oracle
import hold_oracle
import oracle_c
import oracle_py
import remedy_hold_oracle
import timeout_oracle
import window_oracle

KIND_MASK, KIND_INTERVAL, KIND_CRON_SPEC, KIND_CRON_EVERY = 0x7, 2, 3, 4
F_PENDING_OK, F_PENDING_FAIL = 1 << 4, 1 << 5
F_REMEDY_PENDING, F_REMEDY_OUTCOME_OK = 1 << 6, 1 << 7
F_TOMBSTONE = 1 << 8
TZ_SHIFT = 24
CLOSED_LOOP, CATCH_UP = 0x1, 0x8
E_INVAL, E_RANGE = -1, -2
DAY = 86400
NONE = hold_oracle.NOT_IN_FLIGHT
NO_DEADLINE = timeout_oracle.NO_DEADLINE
NO_NEXT = -9223372036 + 1  # RepeatAfterSec when Next() finds nothing (Go zero time)
COLUMN_NAMES = [n for n, _ in oracle_c.COLUMNS]
MASKS = ("minute", "hour", "dom", "month", "dow")
RESULT_STATS = ("n_result_ok", "n_result_fail", "n_remedy_ok", "n_remedy_fail")
NO_TIMEOUTS = (np.zeros(0, dtype=np.uint64), np.zeros(0, dtype=np.int64))
NO_DETAILS = np.zeros(0, dtype=change_details_oracle.DETAIL)

Tick = namedtuple("Tick", "idx act stats timed_out remedy_timed_out")


class Refused(Exception):
    def __init__(self, code):
        super().__init__(code)
        self.code = code


def _last_of(idx):
    """positions of the last occurrence of every distinct slot of idx (a later entry of a call wins)"""
    _, rev = np.unique(idx[::-1], return_index=True)
    return len(idx) - 1 - rev


def _never_matches(c):
    """True when no wall clock in any zone can match the 5-field schedule: an empty field, or no calendar day of
    the next six years (leap years included) that passes the month and day fields"""
    if not (c.minute & ((1 << 60) - 1)) or not (c.hour & ((1 << 24) - 1)) or not (c.month & 0x1FFE):
        return True
    star = (c.dom | c.dow) & oracle_py.STAR_BIT
    for month in range(1, 13):
        if not (c.month >> month & 1):
            continue
        for day in range(1, {2: 29, 4: 30, 6: 30, 9: 30, 11: 30}.get(month, 31) + 1):
            dom_ok = bool(c.dom >> day & 1)
            if star and not dom_ok:
                continue
            if not star and dom_ok:
                return False
            if c.dow & 0x7F:  # some weekday of the six years falls on this date
                return False
    return True


class HandleModel:
    def __init__(self, zmap, capacity, shard_base=0, seed=0, hold=False, remedy=False, track=False, details=False):
        self.zmap = zmap
        self.capacity = capacity
        self.shard_base = shard_base
        self.seed = seed
        self.c = changes_oracle.empty_columns(capacity)
        self.hwm = 0
        self.P = None
        self.since = hold_oracle.none_in_flight(capacity)
        self.wf = np.zeros(capacity, dtype=np.int32)
        self.deadline = timeout_oracle.no_deadlines(capacity)
        self.rsince = hold_oracle.none_in_flight(capacity)
        self.rdeadline = timeout_oracle.no_deadlines(capacity)
        self.hold = self.remedy = self.track = self.details_on = False
        self.hc, self.rm = {}, {}
        self.last = Tick(np.zeros(0, np.uint64), np.zeros(0, np.uint32), None, NO_TIMEOUTS, NO_TIMEOUTS)
        self.changed = changes_oracle.EMPTY
        self.det = NO_DETAILS
        self._opy_ids = {p: oracle_py.tz_lookup(z) for z, p in zmap.ids.items()}
        self._ras_cache = {}
        self.set_hold(hold)
        if remedy:
            self.set_remedy(True)
        self.set_track(track)
        if details:
            self.set_details(True)

    # ---- calls that change state -------------------------------------------------------------------------------
    def _drop(self, slots):
        for i in np.asarray(slots, dtype=np.int64).tolist():
            self.hc.pop(i, None)
            self.rm.pop(i, None)

    def _end_remedy(self, slots):
        self.rsince[slots] = NONE
        self.rdeadline[slots] = NO_DEADLINE

    def upsert(self, idx, recs):
        idx = np.asarray(idx, dtype=np.int64)
        last = _last_of(idx)
        sl = idx[last]
        for name in COLUMN_NAMES:
            self.c[name][sl] = recs[name][last]
        self.c["flags"][sl] &= np.uint32(~F_TOMBSTONE & 0xFFFFFFFF)
        self.wf[sl] = recs["wf_timeout"][last]
        self.hwm = max(self.hwm, int(idx.max()) + 1)
        self._drop(idx)

    def remove(self, idx):
        idx = np.asarray(idx, dtype=np.int64)
        self.c["flags"][idx] = F_TOMBSTONE
        hold_oracle.clear(self.since, idx)
        self.deadline[idx] = NO_DEADLINE
        self._end_remedy(idx)
        self._drop(idx)

    def post(self, idx, phase, rphase=None):
        idx = np.asarray(idx, dtype=np.int64)
        phase = np.asarray(phase, dtype=np.uint8)
        rphase = np.zeros(len(idx), np.uint8) if rphase is None else np.asarray(rphase, dtype=np.uint8)
        if self.details_on:
            v, rv = self.in_flight(idx=idx), self.remedy_in_flight(idx=idx)
            for k, i in enumerate(idx.tolist()):
                if phase[k]:
                    self.hc[i] = int(v[k])
                if rphase[k]:
                    self.rm[i] = int(rv[k])
        f = self.c["flags"]
        for ph, group, bits in ((phase, F_PENDING_OK | F_PENDING_FAIL, {1: F_PENDING_OK, 2: F_PENDING_FAIL}),
                                (rphase, F_REMEDY_PENDING | F_REMEDY_OUTCOME_OK,
                                 {1: F_REMEDY_PENDING | F_REMEDY_OUTCOME_OK, 2: F_REMEDY_PENDING})):
            m = ph != 0
            if m.any():
                last = _last_of(idx[m])
                sl, p = idx[m][last], ph[m][last]
                f[sl] = (f[sl] & np.uint32(~group & 0xFFFFFFFF)) | np.where(p == 1, bits[1], bits[2]).astype(np.uint32)
        hold_oracle.post(self.since, idx, phase)
        self._end_remedy(idx[(phase != 0) | (rphase != 0)])

    def load(self, first, cols):
        n = len(cols["flags"])
        sl = np.arange(first, first + n)
        for name in COLUMN_NAMES:
            self.c[name][first:first + n] = cols[name]
        hold_oracle.clear(self.since, sl)
        self.wf[sl] = 0
        self.deadline[sl] = NO_DEADLINE
        self._end_remedy(sl)
        self.hwm = max(self.hwm, first + n)
        self._drop(sl)

    def read(self, slots=None):
        pass

    def set_hold(self, on):
        if on and not self.hold:
            self.since[:] = NONE
            self.deadline[:] = NO_DEADLINE
        if not on and self.hold:
            self.set_remedy(False)
        self.hold = bool(on)

    def set_remedy(self, on):
        if not self.hold:
            raise Refused(E_INVAL)
        if not on:
            self._end_remedy(slice(None))
        self.remedy = bool(on)

    def set_track(self, on):
        if on and not self.track:
            self.changed = changes_oracle.EMPTY
        if not on:
            self.details_on = False
        self.track = bool(on)

    def set_details(self, on):
        if not self.track:
            raise Refused(E_INVAL)
        if on and not self.details_on:
            self.det = NO_DETAILS  # (the last tick's list has no details)
        self.details_on = bool(on)
        self.hc, self.rm = {}, {}

    # ---- ticks -------------------------------------------------------------------------------------------------
    def view(self):
        """the swept slots' columns (prefix views: the oracles work in place)"""
        return {k: v[:self.hwm] for k, v in self.c.items()}

    def window_of(self, T, mode):
        """P of a catch-up tick at T, or None for a plain one"""
        return self.P if (mode & CATCH_UP) and self.P is not None and T > self.P else None

    def _sweep(self, cols, runs, T, P, mode, seed):
        """the tick path over the swept prefix `cols` and per-slot `runs` (since, D, remedy start, remedy deadline)"""
        since, deadline, rsince, rdeadline = runs
        kw = dict(P=P, shard_base=self.shard_base)
        wf = self.wf[:len(since)]
        if self.remedy:
            return Tick(*remedy_hold_oracle.sweep(self.zmap, cols, since, deadline, wf, rsince, rdeadline, T, **kw))
        if self.hold:
            return Tick(*timeout_oracle.sweep(self.zmap, cols, since, deadline, wf, T, mode=mode & CLOSED_LOOP,
                                              seed=seed, **kw), NO_TIMEOUTS)
        if P is not None:
            out = window_oracle.sweep_window(self.zmap, cols, P, T, mode=mode & CLOSED_LOOP, seed=seed,
                                             shard_base=self.shard_base)
        else:
            out = self.zmap.sweep(cols, T, mode=mode & CLOSED_LOOP, seed=seed, shard_base=self.shard_base)
        return Tick(*out, NO_TIMEOUTS, NO_TIMEOUTS)

    def _runs(self):
        h = self.hwm
        return self.since[:h], self.deadline[:h], self.rsince[:h], self.rdeadline[:h]

    def tick(self, T, mode=0):
        """the tick of every entry point, or Refused"""
        if self.hold and (mode & CLOSED_LOOP):
            raise Refused(E_INVAL)
        P = self.window_of(T, mode)
        if P is not None and T - P > DAY:
            raise Refused(E_RANGE)
        cols = self.view()
        before = changes_oracle.snapshot(cols) if self.track else None
        out = self._sweep(cols, self._runs(), T, P, mode, self.seed)
        self.P = T
        if self.track:
            self.changed = changes_oracle.changed(before, cols, out.idx, out.act, self.shard_base)
        if self.details_on:
            self.det = change_details_oracle.details(self.changed, before["flags"], out, T, mode, self.hc, self.rm,
                                                     self.shard_base)
        self.hc, self.rm = {}, {}
        self.last = out
        return out

    def run_ticks(self, T0, n, mode=0, seed=0):
        """per-tick statistics of am_sweep_run_ticks, or Refused"""
        if self.hold or (mode & CATCH_UP):
            raise Refused(E_INVAL)
        self.seed = seed
        v = self.view()
        rows = [self.zmap.sweep(v, T0 + k, mode=mode & CLOSED_LOOP, seed=seed, shard_base=self.shard_base)[2]
                for k in range(n)]
        self.P = T0 + n - 1
        self.last = self.last._replace(timed_out=NO_TIMEOUTS, remedy_timed_out=NO_TIMEOUTS)
        self.changed, self.det = changes_oracle.EMPTY, NO_DETAILS
        self.hc, self.rm = {}, {}
        return rows

    # ---- queries -----------------------------------------------------------------------------------------------
    def cols(self):
        return self.c

    def _slots(self, first, n, idx):
        if idx is not None:
            return np.asarray(idx, dtype=np.int64)
        return np.arange(first, first + (self.capacity - first if n is None else n))

    def live(self, slots):
        """bool per slot: not a tombstone.  A removed slot's columns other than flags are unspecified until its next
        upsert or load (the handle keeps what the slot held before the drain, the model what it held before the
        remove): compare them for live slots only."""
        return (self.c["flags"][np.asarray(slots, dtype=np.int64)] & np.uint32(F_TOMBSTONE)) == 0

    def in_flight(self, first=0, n=None, idx=None):
        sl = self._slots(first, n, idx)
        if not self.hold:
            return np.full(len(sl), NONE, dtype=np.int64)
        c = {k: self.c[k][sl] for k in ("flags", "finished_at")}
        return hold_oracle.in_flight(c, self.since[sl])

    def remedy_in_flight(self, first=0, n=None, idx=None):
        sl = self._slots(first, n, idx)
        if not self.remedy:
            return np.full(len(sl), NONE, dtype=np.int64)
        return remedy_hold_oracle.in_flight({"flags": self.c["flags"][sl]}, self.rsince[sl])

    def last_timed_out(self):
        return self.last.timed_out

    def last_remedy_timed_out(self):
        return self.last.remedy_timed_out

    def changes(self):
        return self.changed

    def details(self):
        return self.det

    def _zone_repeat_after(self, i, T):
        masks = tuple(int(self.c[k][i]) for k in MASKS)
        tz = self._opy_ids[int(self.c["flags"][i] >> np.uint32(TZ_SHIFT))]
        c = oracle_py.Cron(oracle_py.CRON_SPEC, *masks, tz_id=tz)
        key = (masks, tz, T)
        if key not in self._ras_cache:
            self._ras_cache[key] = NO_NEXT if _never_matches(c) else oracle_py.cron_repeat_after_sec(c, T)
        return self._ras_cache[key]

    def repeat_after(self, T, first, n):
        f = self.c["flags"][first:first + n]
        kind = f & np.uint32(KIND_MASK)
        live = (f & np.uint32(F_TOMBSTONE)) == 0
        out = np.zeros(n, dtype=np.int64)
        iv = live & ((kind == KIND_INTERVAL) | (kind == KIND_CRON_EVERY))
        out[iv] = self.c["ras"][first:first + n][iv]
        lib = oracle_c.load()
        for k in np.flatnonzero(live & (kind == KIND_CRON_SPEC)):
            i = first + int(k)
            if f[k] >> np.uint32(TZ_SHIFT):
                out[k] = self._zone_repeat_after(i, T)
            else:
                c = oracle_c.OrcCron(*(int(self.c[m][i]) for m in MASKS), 0, oracle_py.CRON_SPEC, 0)
                out[k] = lib.orc_cron_repeat_after_sec(C.byref(c), T)
        return out

    def held(self):
        """bool per swept slot: held by the hold or by a remedy run"""
        v, (since, _, rsince, _) = self.view(), self._runs()
        if not self.hold:
            return np.zeros(self.hwm, dtype=bool)
        return hold_oracle.held(v, since) | (remedy_hold_oracle.held(v, rsince) if self.remedy else False)

    def live_zone_schedules(self):
        """live, not held CRON_SPEC records bound to a named zone (am_sweep_next_due only bounds those)"""
        f = self.view()["flags"]
        zc = ((f & np.uint32(KIND_MASK)) == KIND_CRON_SPEC) & ((f >> np.uint32(TZ_SHIFT)) != 0) & \
             ((f & np.uint32(F_TOMBSTONE)) == 0)
        return int((zc & ~self.held()).sum())

    def first_active_tick(self, T, horizon):
        """the first second of (T, T + horizon] at which a plain tick emits anything, applies a posted result or times
        a run of either kind out, by brute force over copies of the state; None when there is none"""
        cols = {k: v.copy() for k, v in self.view().items()}
        runs = tuple(a.copy() for a in self._runs())
        for t in range(T + 1, T + horizon + 1):
            out = self._sweep(cols, runs, t, None, 0, 0)
            if len(out.idx) or len(out.timed_out[0]) or len(out.remedy_timed_out[0]) or \
                    any(out.stats[k] for k in RESULT_STATS):
                return t
        return None
