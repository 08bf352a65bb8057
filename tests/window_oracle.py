"""The oracle of a catch-up tick (AM_SWEEP_CATCH_UP): the C oracle's tick at T with the cron decision replaced by
a brute-force one.  A 5-field schedule is due iff the C oracle's own matches(t) holds at some second t of
(P, T]; everything else is orc_sweep at T.

It shares nothing with the library's calendar boxes:
  * the candidate instants are found one second at a time, per zone, with libc (time.localtime under TZ): every t
    in (P, T] at which the zone's wall clock — UTC's included — shows second 0.  No other second can match
    (ParseStandard pins the Second field to 0);
  * at each candidate t, orc_sweep itself decides which 5-field schedules match: it runs over a probe copy that
    holds only the CRON_SPEC records, stripped of everything but kind and zone (nothing pending, open loop, so a
    probe tick changes nothing and emits exactly the records whose schedule matches at t);
  * the decision is then handed to orc_sweep at T by rewriting the records for that one call: a record that fired
    becomes an interval check that is always due (no repeat timer, RepeatAfterSec = INT32_MIN), one that did not
    keeps a minute mask of zero.  Kind, zone, interval, masks and the caller's timer bit are restored afterwards;
    orc_sweep never writes those columns except to arm the timer when it applies a posted result.
"""
import os
import time

import numpy as np

KIND_MASK, KIND_INTERVAL, KIND_CRON_SPEC = 0x7, 2, 3
F_TOMBSTONE, F_TIMER_ARMED = 1 << 8, 1 << 10
TZ_SHIFT = 24
I32MIN = -(1 << 31)


def minute_starts(zone, P, T):
    """every t in (P, T] at which `zone` (a zone name, or None for UTC) shows second 0, by libc"""
    if zone is None:
        return [t for t in range(P + 1, T + 1) if time.gmtime(t).tm_sec == 0]
    old = os.environ.get("TZ")
    os.environ["TZ"] = ":" + zone
    time.tzset()
    try:
        return [t for t in range(P + 1, T + 1) if time.localtime(t).tm_sec == 0]
    finally:
        if old is None:
            del os.environ["TZ"]
        else:
            os.environ["TZ"] = old
        time.tzset()


def fired_in_window(zmap, ocols, P, T):
    """bool[n]: the record is CRON_SPEC and its schedule matches at some second of (P, T]"""
    flags = ocols["flags"]
    n = len(flags)
    cron = ((flags & np.uint32(KIND_MASK)) == KIND_CRON_SPEC) & ((flags & np.uint32(F_TOMBSTONE)) == 0)
    fired = np.zeros(n, dtype=bool)
    if not cron.any() or T <= P:
        return fired
    names = {v: k for k, v in zmap.ids.items()}
    zones = sorted(set((flags[cron] >> np.uint32(TZ_SHIFT)).tolist()))
    instants = sorted(set(t for z in zones for t in minute_starts(names[z] if z else None, P, T)))
    probe = {k: np.zeros_like(v) for k, v in ocols.items()}
    for k in ("minute", "hour", "dom", "month", "dow"):
        probe[k][:] = ocols[k]
    probe["flags"][:] = np.where(cron, flags & np.uint32(KIND_MASK | (0xFF << TZ_SHIFT)), np.uint32(F_TOMBSTONE))
    for t in instants:
        idx, _, _ = zmap.sweep(probe, t)
        fired[idx.astype(np.int64)] = True
    return fired


def sweep_window(zmap, ocols, P, T, mode=0, seed=0, shard_base=0):
    """orc_sweep_window: the catch-up tick at T after a previous tick at P, over numpy SoA columns that carry the
    product's zone ids, IN PLACE.  Returns (global idx, action, stats) like oracle_c.sweep."""
    flags0 = ocols["flags"].copy()
    ras0 = ocols["ras"].copy()
    minute0 = ocols["minute"].copy()
    cron = ((flags0 & np.uint32(KIND_MASK)) == KIND_CRON_SPEC) & ((flags0 & np.uint32(F_TOMBSTONE)) == 0)
    fired = fired_in_window(zmap, ocols, P, T)
    keep = np.uint32(~(KIND_MASK | F_TIMER_ARMED | (0xFF << TZ_SHIFT)) & 0xFFFFFFFF)
    ocols["flags"][fired] = (flags0[fired] & keep) | np.uint32(KIND_INTERVAL)
    ocols["ras"][fired] = I32MIN
    ocols["minute"][cron & ~fired] = 0
    try:
        return zmap.sweep(ocols, T, mode=mode & 1, seed=seed, shard_base=shard_base)
    finally:
        ocols["ras"][:] = ras0
        ocols["minute"][:] = minute0
        back = np.uint32(KIND_MASK | (0xFF << TZ_SHIFT))
        f = ocols["flags"]
        f[cron] = (f[cron] & ~back) | (flags0[cron] & back) | (flags0[cron] & np.uint32(F_TIMER_ARMED))
