"""The oracle of a tick under a submit budget (am_sweep_set_submit_budget, DESIGN §6 item 19), composed of the per-tick
oracles: the unlimited tick (hold_oracle / timeout_oracle / remedy_hold_oracle through tests/handle_model.py) with the
checks that wait for admission forced due, then the cut.

`wait[i]` is the second since which slot i waits for admission, or NOT_WAITING.  For one tick at T:
  1. every waiting slot that is a candidate whatever its schedule — live, INTERVAL / CRON_EVERY / CRON_SPEC, not held —
     is rewritten for the call so that the tick finds it due, as tests/window_oracle.py rewrites the records that fired:
     an interval check without a repeat timer and RepeatAfterSec = INT32_MIN, zone bits cleared.  Kind, zone, interval
     are restored afterwards and the timer bit ORed back (`force_due`, `restore`); nothing after the due decision depends on them;
  2. the unlimited tick runs;
  3. `cut`: the candidates are its entries with SUBMIT_HC.  Waiting ones by (wait, slot), then fresh ones by slot; the
     first `budget` are admitted (their wait ends), the others lose SUBMIT_HC (an entry with nothing left leaves the
     list), their since and deadline become none and they wait from T on unless they already did.  A slot that waited
     and is not a candidate stops waiting.  The statistics follow the trimmed list; the result counters do not change.
"""
import numpy as np

KIND_MASK, KIND_INTERVAL, KIND_CRON_SPEC, KIND_CRON_EVERY = 0x7, 2, 3, 4
F_TOMBSTONE, F_TIMER_ARMED = 1 << 8, 1 << 10
TZ_SHIFT = 24
I32MIN = -(1 << 31)
ACT_SUBMIT_HC = 0x01
NOT_WAITING = -(1 << 63)
NO_DEADLINE = (1 << 63) - 1
UNLIMITED = (1 << 64) - 1
INT64_MAX = (1 << 63) - 1
U64 = np.uint64


def can_be_due(flags):
    kind = flags & np.uint32(KIND_MASK)
    live = ((flags & np.uint32(F_TOMBSTONE)) == 0) & (kind >= 1) & (kind <= 5)
    return live & ((kind == KIND_INTERVAL) | (kind == KIND_CRON_EVERY) | (kind == KIND_CRON_SPEC))


def force_due(ocols, slots):
    """step 1, IN PLACE on the columns; returns what `restore` needs"""
    saved = {k: ocols[k][slots].copy() for k in ("flags", "ras")}
    keep = np.uint32(~(KIND_MASK | F_TIMER_ARMED | (0xFF << TZ_SHIFT)) & 0xFFFFFFFF)
    ocols["flags"][slots] = (saved["flags"] & keep) | np.uint32(KIND_INTERVAL)
    ocols["ras"][slots] = I32MIN
    return slots, saved


def restore(ocols, forced):
    slots, saved = forced
    ocols["ras"][slots] = saved["ras"]
    back = np.uint32(KIND_MASK | (0xFF << TZ_SHIFT))  # (a result the tick applied may have armed the timer)
    f = ocols["flags"]
    f[slots] = (f[slots] & ~back) | (saved["flags"] & (back | np.uint32(F_TIMER_ARMED)))


def empty_admission():
    return {"n_candidates": 0, "n_admitted": 0, "n_deferred": 0, "oldest_deferred": INT64_MAX}


def cut(idx, act, stats, wait, since, deadline, budget, T, shard_base=0):
    """step 3 on the unlimited tick's (global idx, act, stats), IN PLACE on wait / since / deadline (local slots, the
    swept prefix).  Returns (idx, act, stats, admission)."""
    idx = np.asarray(idx, dtype=np.uint64)
    act = np.asarray(act, dtype=np.uint32).copy()
    loc = idx.astype(np.int64) - int(shard_base)
    sub = (act & ACT_SUBMIT_HC) != 0
    cand = loc[sub]
    waiting = wait[cand] != NOT_WAITING
    w = cand[waiting]
    w = w[np.lexsort((w, wait[w]))]
    queue = np.concatenate([w, cand[~waiting]])
    n_adm = min(budget, len(queue))
    admitted, deferred = queue[:n_adm], queue[n_adm:]
    ended = np.ones(len(wait), dtype=bool)
    ended[cand] = False
    wait[ended] = NOT_WAITING
    wait[admitted] = NOT_WAITING
    wait[deferred[wait[deferred] == NOT_WAITING]] = T
    since[deferred] = NOT_WAITING
    deadline[deferred] = NO_DEADLINE
    trimmed = np.zeros(len(wait), dtype=bool)
    trimmed[deferred] = True
    hit = np.zeros(len(loc), dtype=bool)
    hit[sub] = trimmed[cand]
    act[hit] &= np.uint32(~ACT_SUBMIT_HC & 0xFFFFFFFF)
    keep = act != 0
    idx, act = idx[keep], act[keep]
    st = dict(stats)
    st["n_emitted"] = len(idx)
    st["n_submit_hc"] -= len(deferred)
    st["idx_xor"] = int(np.bitwise_xor.reduce(idx)) if len(idx) else 0
    st["idx_sum"] = int(idx.sum(dtype=U64)) if len(idx) else 0
    left = wait[wait != NOT_WAITING]
    adm = {"n_candidates": len(queue), "n_admitted": n_adm, "n_deferred": len(left),
           "oldest_deferred": int(left.min()) if len(left) else INT64_MAX}
    return idx, act, st, adm
