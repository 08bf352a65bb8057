"""One sequential model of a sweep handle, built only from the existing oracles, for random call sequences through
every entry point (tests/test_call_sequences_gpu.py).

The model holds what the handle holds: the sixteen columns of every slot (in the product's zone ids, like
adversarial.ZoneMap), the hold's `since` per slot and whether the hold is on, the previous tick's second P and the
high-water mark of the swept slots.  Every library call has a method; calls apply in call order (DESIGN §6 item 9):
  * upsert / remove / post / load change the columns at once (a posted phase sets the pending bits the next tick
    applies, so a later upsert or load of the slot supersedes it; a workflow phase, a remove and a load clear since);
  * a tick is zmap.sweep over the swept slots; a catch-up tick (P set and T > P) is window_oracle.sweep_window; a tick
    with the hold on is hold_oracle.sweep (around either);
  * a refused call raises Refused and changes nothing.  P follows DESIGN §6 item 11: every successful tick sets it,
    one that returns AM_E_NOSPACE included; run_ticks sets it to its last second; AM_E_RANGE / AM_E_INVAL refusals
    leave it;
  * the queries: repeat_after (interval and "@every": the stored interval; a UTC 5-field schedule: the C oracle's
    orc_cron_repeat_after_sec; one bound to a named zone: the Python oracle's "first instant whose wall clock
    matches", DESIGN §6 item 10; everything else, tombstones included, 0), next_due_bound (the first plain tick that
    does anything, by brute force over copies) and in_flight (hold_oracle.in_flight)."""
import ctypes as C

import numpy as np

import hold_oracle
import oracle_c
import oracle_py
import window_oracle

KIND_MASK, KIND_INTERVAL, KIND_CRON_SPEC, KIND_CRON_EVERY = 0x7, 2, 3, 4
F_PENDING_OK, F_PENDING_FAIL = 1 << 4, 1 << 5
F_REMEDY_PENDING, F_REMEDY_OUTCOME_OK = 1 << 6, 1 << 7
F_TOMBSTONE = 1 << 8
TZ_SHIFT = 24
CLOSED_LOOP, CATCH_UP = 0x1, 0x8
E_INVAL, E_RANGE = -1, -2
NONE = hold_oracle.NOT_IN_FLIGHT
NO_NEXT = -9223372036 + 1  # RepeatAfterSec when Next() finds nothing (Go zero time)
COLUMN_NAMES = [n for n, _ in oracle_c.COLUMNS]
MASKS = ("minute", "hour", "dom", "month", "dow")
RESULT_STATS = ("n_result_ok", "n_result_fail", "n_remedy_ok", "n_remedy_fail")


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


class SequenceModel:
    def __init__(self, zmap, capacity, shard_base=0, seed=0):
        self.zmap = zmap
        self.capacity = capacity
        self.shard_base = shard_base
        self.seed = seed
        self.cols = {n: np.zeros(capacity, dtype=dt) for n, dt in oracle_c.COLUMNS}
        self.cols["flags"][:] = F_TOMBSTONE
        self.since = hold_oracle.none_in_flight(capacity)
        self.hold = False
        self.P = None
        self.hwm = 0
        self._opy_ids = {p: oracle_py.tz_lookup(z) for z, p in zmap.ids.items()}
        self._ras_cache = {}

    # ---- calls that change state -------------------------------------------------------------------------------
    def upsert(self, idx, recs):
        idx = np.asarray(idx, dtype=np.int64)
        last = _last_of(idx)
        sl = idx[last]
        for name in COLUMN_NAMES:
            self.cols[name][sl] = recs[name][last]
        self.cols["flags"][sl] &= np.uint32(~F_TOMBSTONE & 0xFFFFFFFF)
        self.hwm = max(self.hwm, int(idx.max()) + 1)

    def remove(self, idx):
        idx = np.asarray(idx, dtype=np.int64)
        self.cols["flags"][idx] = F_TOMBSTONE
        hold_oracle.clear(self.since, idx)

    def post(self, idx, phase, rphase=None):
        idx = np.asarray(idx, dtype=np.int64)
        phase = np.asarray(phase, dtype=np.uint8)
        f = self.cols["flags"]
        hc, rm = np.uint32(F_PENDING_OK | F_PENDING_FAIL), np.uint32(F_REMEDY_PENDING | F_REMEDY_OUTCOME_OK)
        m = phase != 0
        if m.any():
            last = _last_of(idx[m])
            sl, ph = idx[m][last], phase[m][last]
            f[sl] = (f[sl] & ~hc) | np.where(ph == 1, F_PENDING_OK, F_PENDING_FAIL).astype(np.uint32)
        if rphase is not None:
            rphase = np.asarray(rphase, dtype=np.uint8)
            m = rphase != 0
            if m.any():
                last = _last_of(idx[m])
                sl, ph = idx[m][last], rphase[m][last]
                f[sl] = (f[sl] & ~rm) | np.where(ph == 1, rm, np.uint32(F_REMEDY_PENDING)).astype(np.uint32)
        hold_oracle.post(self.since, idx, phase)

    def load(self, first, cols):
        n = len(cols["flags"])
        for name in COLUMN_NAMES:
            self.cols[name][first:first + n] = cols[name]
        hold_oracle.clear(self.since, np.arange(first, first + n))
        self.hwm = max(self.hwm, first + n)

    def set_hold(self, on):
        if on and not self.hold:
            self.since[:] = NONE
        self.hold = bool(on)

    # ---- ticks -------------------------------------------------------------------------------------------------
    def view(self):
        """the swept slots' columns (prefix views: the oracles work in place)"""
        return {k: v[:self.hwm] for k, v in self.cols.items()}

    def window_of(self, T, mode):
        """P of a catch-up tick at T, or None for a plain one"""
        return self.P if (mode & CATCH_UP) and self.P is not None and T > self.P else None

    def _sweep(self, cols, since, T, P, mode, seed):
        if self.hold:
            return hold_oracle.sweep(self.zmap, cols, since, T, P=P, mode=mode & CLOSED_LOOP, seed=seed,
                                     shard_base=self.shard_base)
        if P is not None:
            return window_oracle.sweep_window(self.zmap, cols, P, T, mode=mode & CLOSED_LOOP, seed=seed,
                                              shard_base=self.shard_base)
        return self.zmap.sweep(cols, T, mode=mode & CLOSED_LOOP, seed=seed, shard_base=self.shard_base)

    def tick(self, T, mode):
        """the tick of every entry point: (global idx, action, stats), or Refused"""
        if self.hold and (mode & CLOSED_LOOP):
            raise Refused(E_INVAL)
        P = self.window_of(T, mode)
        if P is not None and T - P > 86400:
            raise Refused(E_RANGE)
        out = self._sweep(self.view(), self.since[:self.hwm], T, P, mode, self.seed)
        self.P = T
        return out

    def run_ticks(self, T0, n, mode, seed):
        """per-tick statistics of am_sweep_run_ticks, or Refused"""
        if self.hold or (mode & CATCH_UP):
            raise Refused(E_INVAL)
        self.seed = seed
        v = self.view()
        rows = [self.zmap.sweep(v, T0 + k, mode=mode & CLOSED_LOOP, seed=seed, shard_base=self.shard_base)[2]
                for k in range(n)]
        self.P = T0 + n - 1
        return rows

    # ---- queries -----------------------------------------------------------------------------------------------
    def live(self, slots):
        """bool per slot: not a tombstone.  A removed slot's columns other than flags are unspecified until its next
        upsert or load (the handle keeps what the slot held before the drain, the model what it held before the
        remove): compare them for live slots only."""
        return (self.cols["flags"][np.asarray(slots, dtype=np.int64)] & np.uint32(F_TOMBSTONE)) == 0

    def in_flight(self, first=0, n=None, idx=None):
        sl = np.asarray(idx, dtype=np.int64) if idx is not None else np.arange(first, first + n)
        if not self.hold:
            return np.full(len(sl), NONE, dtype=np.int64)
        c = {k: self.cols[k][sl] for k in ("flags", "finished_at")}
        return hold_oracle.in_flight(c, self.since[sl])

    def _zone_repeat_after(self, i, T):
        masks = tuple(int(self.cols[k][i]) for k in MASKS)
        tz = self._opy_ids[int(self.cols["flags"][i] >> np.uint32(TZ_SHIFT))]
        c = oracle_py.Cron(oracle_py.CRON_SPEC, *masks, tz_id=tz)
        key = (masks, tz, T)
        if key not in self._ras_cache:
            self._ras_cache[key] = NO_NEXT if _never_matches(c) else oracle_py.cron_repeat_after_sec(c, T)
        return self._ras_cache[key]

    def repeat_after(self, T, first, n):
        f = self.cols["flags"][first:first + n]
        kind = f & np.uint32(KIND_MASK)
        live = (f & np.uint32(F_TOMBSTONE)) == 0
        out = np.zeros(n, dtype=np.int64)
        iv = live & ((kind == KIND_INTERVAL) | (kind == KIND_CRON_EVERY))
        out[iv] = self.cols["ras"][first:first + n][iv]
        lib = oracle_c.load()
        for k in np.flatnonzero(live & (kind == KIND_CRON_SPEC)):
            i = first + int(k)
            if f[k] >> np.uint32(TZ_SHIFT):
                out[k] = self._zone_repeat_after(i, T)
            else:
                c = oracle_c.OrcCron(*(int(self.cols[m][i]) for m in MASKS), 0, oracle_py.CRON_SPEC, 0)
                out[k] = lib.orc_cron_repeat_after_sec(C.byref(c), T)
        return out

    def live_zone_schedules(self):
        """live, not held CRON_SPEC records bound to a named zone (am_sweep_next_due only bounds those)"""
        v = self.view()
        f = v["flags"]
        zc = ((f & np.uint32(KIND_MASK)) == KIND_CRON_SPEC) & ((f >> np.uint32(TZ_SHIFT)) != 0) & \
             ((f & np.uint32(F_TOMBSTONE)) == 0)
        if self.hold:
            zc &= ~hold_oracle.held(v, self.since[:self.hwm])
        return int(zc.sum())

    def first_active_tick(self, T, horizon):
        """the first second of (T, T + horizon] at which a plain tick emits anything or applies a posted result, by
        brute force over copies of the state; None when there is none"""
        cols = {k: v.copy() for k, v in self.view().items()}
        since = self.since[:self.hwm].copy()
        for t in range(T + 1, T + horizon + 1):
            _, _, st = self._sweep(cols, since, t, None, 0, 0)
            if st["n_emitted"] or any(st[k] for k in RESULT_STATS):
                return t
        return None
