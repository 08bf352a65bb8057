"""The changed set of a tick (am_sweep_set_track_changes / am_sweep_last_changes), defined from the existing oracles'
states alone: the slots whose sixteen columns differ between the state just before the tick (every call before it
applied, as the oracles apply them) and the state after it.  Two groups of flag bits do not count: the library-internal
carry bits (AM_F_CARRY_MASK) and the posted-result bits AM_F_PENDING_* / AM_F_REMEDY_* that the tick consumes.  The
records whose action carries AM_ACT_ANOMALY without AM_ACT_STOPPED are taken out: the reference panics at hcc.go:690
before it writes a status (DESIGN.md section 6 item 5), although the oracles count the Failed.

The states come from tests/handle_model.py.  Nothing is taken from the device's mechanism (drain marks, exceptions,
bitmaps)."""
import numpy as np

import oracle_c

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
