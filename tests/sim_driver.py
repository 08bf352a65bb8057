"""The oracle of am_sweep_simulate: the loop its contract states, driven on tests/handle_model.py's HandleModel with both
holds on.  Per tick T it posts, through model.post, the phase of every held health-check run (model.in_flight) and of
every held remedy run (model.remedy_in_flight) whose simulated end is <= T, then ticks the model at T.  The draws are
the contract's, in numpy: k = the closed loop's keyed splitmix64 of (seed, global index, start); a health-check run
fails iff (k & 0xFF) < the record's fail_p8 and lasts wf_min + (k >> 32) % (wf_max - wf_min + 1) seconds; a remedy run
succeeds iff ((k >> 8) & 0xFF) < 179 and lasts remedy_min + (k >> 32) % (remedy_max - remedy_min + 1) seconds.
Nothing here decides anything the model does not."""
import numpy as np

import changes_oracle
from handle_model import E_INVAL, E_RANGE, NO_DETAILS, NO_TIMEOUTS, NONE, Refused

FULL_SCAN, BLOCKED = 0x2, 0x4
PHASE_OK, PHASE_FAILED = 1, 2
M = np.uint64


def _sm64(z):
    with np.errstate(over="ignore"):
        z = z + M(0x9E3779B97F4A7C15)
        z = (z ^ (z >> M(30))) * M(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> M(27))) * M(0x94D049BB133111EB)
        return z ^ (z >> M(31))


def outcome_key(seed, g, start):
    """the closed loop's key of (seed, global index, second), vectorised over g and start"""
    with np.errstate(over="ignore"):
        return _sm64(_sm64(M(seed) ^ _sm64(np.asarray(g, dtype=M))) + np.asarray(start, dtype=np.int64).view(M))


def draw(seed, g, start, params, failp8=None):
    """(end second, phase) of runs started at `start`: health-check runs with `failp8`, remedy runs without"""
    wf_min, wf_max, r_min, r_max = params
    k = outcome_key(seed, g, start)
    lo, span = (wf_min, wf_max - wf_min + 1) if failp8 is not None else (r_min, r_max - r_min + 1)
    end = np.asarray(start, dtype=np.int64) + lo + ((k >> M(32)) % M(span)).astype(np.int64)
    if failp8 is not None:
        phase = np.where((k & M(0xFF)) < np.asarray(failp8, dtype=M), PHASE_FAILED, PHASE_OK)
    else:
        phase = np.where(((k >> M(8)) & M(0xFF)) < M(179), PHASE_OK, PHASE_FAILED)
    return end, phase.astype(np.uint8)


def refusal(m, T0, n, mode, params):
    """the code am_sweep_simulate refuses with, or None"""
    if params is None or mode & ~(FULL_SCAN | BLOCKED) or n > 1 << 24:
        return E_INVAL
    wf_min, wf_max, r_min, r_max = params
    if wf_min < 1 or wf_max < wf_min or r_min < 1 or r_max < r_min:
        return E_INVAL
    if not (-(1 << 55) < T0 < 1 << 55 and -(1 << 55) < T0 + n < 1 << 55):
        return E_RANGE
    if not (m.hold and m.remedy):
        return E_INVAL
    return None


def simulate(m, T0, n, mode, seed, params):
    """am_sweep_simulate on the model: (stats rows as dicts, sim rows as (in flight, remedy in flight, timed out,
    remedy timed out)), or Refused"""
    code = refusal(m, T0, n, mode, params)
    if code is not None:
        raise Refused(code)
    if n == 0:
        return [], []
    m.seed = seed
    rows, sims = [], []
    g0 = np.uint64(m.shard_base)
    for k in range(n):
        T = T0 + k
        since = m.in_flight(0, m.hwm)
        sl = np.flatnonzero(since != NONE)
        if len(sl):
            failp8 = (m.c["flags"][sl] >> np.uint32(16)) & np.uint32(0xFF)
            end, phase = draw(seed, sl.astype(np.uint64) + g0, since[sl], params, failp8)
            done = end <= T
            if done.any():
                m.post(sl[done], phase[done])
        rsince = m.remedy_in_flight(0, m.hwm)
        rsl = np.flatnonzero(rsince != NONE)
        if len(rsl):
            end, rphase = draw(seed, rsl.astype(np.uint64) + g0, rsince[rsl], params)
            done = end <= T
            if done.any():
                m.post(rsl[done], np.zeros(int(done.sum()), np.uint8), rphase[done])
        out = m.tick(T, mode & FULL_SCAN)
        rows.append(out.stats)
        sims.append((int((m.in_flight(0, m.hwm) != NONE).sum()), int((m.remedy_in_flight(0, m.hwm) != NONE).sum()),
                     len(out.timed_out[0]), len(out.remedy_timed_out[0])))
    # no per-tick lists: the timed-out lists and the change list are empty afterwards
    m.last = m.last._replace(timed_out=NO_TIMEOUTS, remedy_timed_out=NO_TIMEOUTS)
    m.changed, m.det = changes_oracle.EMPTY, NO_DETAILS
    m.hc, m.rm = {}, {}
    return rows, sims
