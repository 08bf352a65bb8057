"""The changed set of a tick (am_sweep_set_track_changes / am_sweep_last_changes), defined from the existing oracles'
states alone: the slots whose sixteen columns differ between the state just before the tick (every call before it
applied, as the oracles apply them) and the state after it.  Two groups of flag bits do not count: the library-internal
carry bits (AM_F_CARRY_MASK) and the posted-result bits AM_F_PENDING_* / AM_F_REMEDY_* that the tick consumes.  The
records whose action carries AM_ACT_ANOMALY without AM_ACT_STOPPED are taken out: the reference panics at hcc.go:690
before it writes a status (DESIGN.md section 6 item 5), although the oracles count the Failed.

The states come from sequence_model.SequenceModel (plain ticks, catch-up ticks, closed loop, the hold in flight) or
remedy_hold_oracle.State (the hold with workflow timeouts and the remedy hold).  Nothing is taken from the device's
mechanism (drain marks, exceptions, bitmaps)."""
import numpy as np

import oracle_c
import remedy_hold_oracle
from sequence_model import SequenceModel

COLUMN_NAMES = [n for n, _ in oracle_c.COLUMNS]
F_RESULT_BITS = (1 << 4) | (1 << 5) | (1 << 6) | (1 << 7)
F_CARRY_MASK = 0x1F << 11
F_TOMBSTONE = 1 << 8
KEEP = np.uint32(~(F_RESULT_BITS | F_CARRY_MASK) & 0xFFFFFFFF)
ACT_STOPPED, ACT_ANOMALY = 0x04, 0x80
EMPTY = np.zeros(0, dtype=np.uint64)


def snapshot(cols):
    return {k: np.array(v, copy=True) for k, v in cols.items()}


def changed(before, after, idx, act, shard_base=0):
    """global indices (ascending u64) of the slots a tick changed: `before` / `after` are the columns around the tick,
    (idx, act) its list"""
    n = len(after["flags"])
    diff = np.zeros(n, dtype=bool)
    for name in COLUMN_NAMES:
        a, b = before[name][:n], after[name][:n]
        if name == "flags":
            a, b = a & KEEP, b & KEEP
        diff |= a != b
    loc = np.asarray(idx, dtype=np.int64) - int(shard_base)
    act = np.asarray(act, dtype=np.uint32)
    diff[loc[((act & ACT_ANOMALY) != 0) & ((act & ACT_STOPPED) == 0)]] = False
    return np.flatnonzero(diff).astype(np.uint64) + np.uint64(shard_base)


def empty_columns(n):
    cols = {name: np.zeros(n, dtype=dt) for name, dt in oracle_c.COLUMNS}
    cols["flags"][:] = F_TOMBSTONE
    return cols


class Model:
    """one oracle state and the changed set of its last tick.  hold: None (off), "hold" (the hold in flight) or
    "remedy" (the hold, workflow timeouts and the remedy hold).  Calls as the models have them; a read drains on the
    handle and changes nothing here."""

    def __init__(self, zmap, n, hold=None, shard_base=0, seed=0):
        self.hold, self.n, self.shard_base = hold, n, shard_base
        if hold == "remedy":
            self.m = remedy_hold_oracle.State(zmap, empty_columns(n), shard_base)
        else:
            self.m = SequenceModel(zmap, n, shard_base, seed=seed)
            self.m.set_hold(hold == "hold")
        self.last = EMPTY

    @property
    def cols(self):
        return self.m.ocols if self.hold == "remedy" else self.m.cols

    def upsert(self, slots, recs):
        self.m.upsert(slots, recs)

    def remove(self, slots):
        self.m.remove(slots)

    def post(self, slots, phase, rphase=None):
        self.m.post(slots, phase, rphase)

    def load(self, first, cols):
        self.m.load(first, cols)

    def read(self, slots):
        pass

    def tick(self, T, mode=0):
        """the oracle's tick: (global idx, action, stats[, timed-out, remedy timed-out])"""
        before = snapshot(self.cols)
        out = self.m.tick(T, mode)
        self.last = changed(before, self.cols, out[0], out[1], self.shard_base)
        return out

    def run_ticks(self, T0, n, mode=0, seed=0):
        """am_sweep_run_ticks: it tracks nothing and empties the list"""
        rows = self.m.run_ticks(T0, n, mode, seed)
        self.last = EMPTY
        return rows

    def changes(self):
        return self.last
