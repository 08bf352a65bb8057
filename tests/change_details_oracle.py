"""The change details of a tick (am_sweep_set_change_details / am_sweep_last_change_details), defined from the existing
models alone, around changes_oracle.changed (which gives the listed slots); tests/handle_model.py takes the starts:

  applied         the posted-result bits of the state just before the tick (every call before it applied, as the
                  models apply them) that the tick consumed, as AM_CHG_* bits; plus FAILED | TIMED_OUT for a slot in
                  the tick's timed-out list, REMEDY_FAILED | REMEDY_TIMED_OUT for one in its remedy timed-out list,
                  STOPPED for an entry reported AM_ACT_STOPPED and CLOSED_LOOP for one emitted with AM_ACT_SUBMIT_HC by
                  a closed-loop tick.
  started         the model's own in_flight() for the slot, taken just before the post call that staged the pending
                  workflow phase (a wrapper around post, before it delegates); the timed-out run's start for a
                  timeout; T for a closed-loop completion; else INT64_MIN.
  remedy_started  the same with remedy_in_flight() (the remedy hold) and the remedy phase; else INT64_MIN.
  action          the slot's action in the tick's list, 0 when it has none.

An upsert, remove or load of a slot drops what was taken for it (its pending phases are gone); a tick drops everything
(it consumes every pending result of a live record, and only live records are listed).  Nothing is taken while details
are off, and turning them on drops everything: results pending from before report INT64_MIN.  Nothing is taken from
the device's mechanism (drain marks, since words, call tags)."""
import numpy as np

NONE = np.int64(np.iinfo(np.int64).min)
F_PENDING_OK, F_PENDING_FAIL, F_REMEDY_PENDING, F_REMEDY_OUTCOME_OK = 1 << 4, 1 << 5, 1 << 6, 1 << 7
CHG_SUCCEEDED, CHG_FAILED, CHG_TIMED_OUT, CHG_REMEDY_SUCCEEDED = 0x01, 0x02, 0x04, 0x08
CHG_REMEDY_FAILED, CHG_REMEDY_TIMED_OUT, CHG_STOPPED, CHG_CLOSED_LOOP = 0x10, 0x20, 0x40, 0x80
ACT_SUBMIT_HC, ACT_STOPPED = 0x01, 0x04
CLOSED = 0x1
DETAIL = np.dtype([("started", "<i8"), ("remedy_started", "<i8"), ("applied", "<u4"), ("action", "<u4")])


def applied_of(f):
    """AM_CHG_* bits of flags words' posted-result bits"""
    f = np.asarray(f, dtype=np.uint32)
    a = np.where(f & F_PENDING_OK, CHG_SUCCEEDED, 0) | np.where(f & F_PENDING_FAIL, CHG_FAILED, 0)
    rem = (f & F_REMEDY_PENDING) != 0
    a |= np.where(rem, np.where(f & F_REMEDY_OUTCOME_OK, CHG_REMEDY_SUCCEEDED, CHG_REMEDY_FAILED), 0)
    return a.astype(np.uint32)


def _lookup(keys, vals, listed, default):
    """vals[keys == listed[k]] per k (default where absent); keys need not be sorted"""
    keys = np.asarray(keys, dtype=np.uint64)
    vals = np.asarray(vals)
    out = np.full(len(listed), default, dtype=np.int64)
    if len(keys) == 0 or len(listed) == 0:
        return out, np.zeros(len(listed), bool)
    order = np.argsort(keys, kind="stable")
    ks, vs = keys[order], vals[order]
    pos = np.minimum(np.searchsorted(ks, listed), len(ks) - 1)
    hit = ks[pos] == listed
    out[hit] = vs[pos[hit]]
    return out, hit


def details(listed, before_flags, out, T, mode, hc, rm, shard_base=0):
    """the details of the listed slots (global idx, ascending) of a tick: `before_flags` the flags before it, `out` its
    oracle output, hc / rm the starts taken at the posts {local slot: start}"""
    listed = np.asarray(listed, dtype=np.uint64)
    loc = (listed - np.uint64(shard_base)).astype(np.int64)
    a = applied_of(np.asarray(before_flags)[loc]).astype(np.int64)
    n = len(before_flags)
    hs, rs = np.full(n, NONE, np.int64), np.full(n, NONE, np.int64)
    for i, v in hc.items():
        hs[i] = v
    for i, v in rm.items():
        rs[i] = v
    st = np.where(a & (CHG_SUCCEEDED | CHG_FAILED), hs[loc], NONE)
    rst = np.where(a & (CHG_REMEDY_SUCCEEDED | CHG_REMEDY_FAILED), rs[loc], NONE)
    act, _ = _lookup(out[0], np.asarray(out[1], dtype=np.int64), listed, 0)
    if len(out) > 3:
        v, hit = _lookup(out[3][0], out[3][1], listed, NONE)
        a |= np.where(hit, CHG_FAILED | CHG_TIMED_OUT, 0)
        st = np.where(hit, v, st)
    if len(out) > 4:
        v, hit = _lookup(out[4][0], out[4][1], listed, NONE)
        a |= np.where(hit, CHG_REMEDY_FAILED | CHG_REMEDY_TIMED_OUT, 0)
        rst = np.where(hit, v, rst)
    a |= np.where(act & ACT_STOPPED, CHG_STOPPED, 0)
    closed = ((act & ACT_SUBMIT_HC) != 0) & bool(mode & CLOSED)
    a |= np.where(closed, CHG_CLOSED_LOOP, 0)
    st = np.where(closed, np.int64(T), st)
    d = np.zeros(len(listed), dtype=DETAIL)
    d["started"], d["remedy_started"], d["applied"], d["action"] = st, rst, a, act
    return d
