"""Hand-derived cases of the status changes (am_sweep_set_track_changes), written against a driver: the oracle alone
(tests/handle_model.py, tests/test_changes_oracle.py) or a handle compared with it after every tick
(tests/test_status_changes_gpu.py, through every tick entry point).  A driver has upsert, remove, post, read(slots),
tick(T, mode=0) -> (global idx, action, stats, ...) and changes() -> the last tick's changed set (global idx).  Each case
names the hold it needs in its `hold` attribute (None, "hold" or "remedy": the hold with timeouts and the remedy
hold) and the capacity in `n`."""
import numpy as np

from timeout_cases import M0, _acts, _timed, rec

OK, FAIL, NONE_PHASE = 1, 2, 0
ANOMALY, STOPPED = 0x80, 0x04


def _ch(d):
    return np.asarray(d.changes()).tolist()


def _case(hold=None, n=8):
    def wrap(f):
        f.hold, f.n = hold, n
        return f
    return wrap


def _interval(am, k, has_remedy=False, W=0, ras=60, age=10):
    return np.concatenate([rec(am, W, repeat_after_sec=ras, finished_at=M0 - age, has_remedy=has_remedy)] * k)


@_case()
def success_without_reset(am, d):
    """a Succeeded on a check without a remedy reset changes SuccessCount, finishedAt and the timer but emits nothing"""
    d.upsert([0, 1], _interval(am, 2))
    d.tick(M0)
    assert _ch(d) == []
    d.post([0], [OK])
    out = d.tick(M0 + 1)
    assert len(out[0]) == 0 and _ch(d) == [0]
    d.tick(M0 + 2)
    assert _ch(d) == []


@_case()
def remedy_phase_alone(am, d):
    """a remedy phase posted on its own changes the remedy counters and emits nothing"""
    d.upsert([0, 1], _interval(am, 2, has_remedy=True))
    d.post([1], [NONE_PHASE], [FAIL])
    out = d.tick(M0)
    assert len(out[0]) == 0 and _ch(d) == [1]


@_case()
def superseded_result(am, d):
    """a result followed by an upsert of its slot is not applied; a result posted after the upsert is"""
    d.upsert([0, 1, 2], _interval(am, 3))
    d.post([0, 1, 2], [FAIL, FAIL, FAIL])
    d.upsert([0, 2], _interval(am, 2))
    d.post([2], [OK])
    d.tick(M0)
    assert _ch(d) == [1, 2]


@_case()
def result_on_removed_slot(am, d):
    """a result on a slot removed after it, or posted to a removed slot, changes nothing"""
    d.upsert([0, 1, 2], _interval(am, 3))
    d.post([0], [OK])
    d.remove([0, 1])
    d.post([1], [FAIL])
    d.post([2], [FAIL])
    d.tick(M0)
    assert _ch(d) == [2]


@_case()
def anomaly(am, d):
    """a Failed that hits the nil-RemedyFinishedAt case is reported AM_ACT_ANOMALY and not listed, although FailedCount
    moves (the reference panics before it writes a status)"""
    d.upsert([0, 1], np.concatenate([rec(am, 0, repeat_after_sec=60, finished_at=M0 - 10, has_remedy=True,
                                         remedy_runs_limit=1, remedy_reset_interval=60, remedy_total_runs=1)] * 2))
    d.post([0, 1], [FAIL, OK])
    out = d.tick(M0)
    assert _acts(out).get(0, 0) & ANOMALY and _ch(d) == [1]


@_case()
def stopped_once(am, d):
    """a stopped check is listed at the tick that reports it, and not again"""
    d.upsert([3], rec(am, 0, repeat_after_sec=0))
    out = d.tick(M0)
    assert _acts(out) == {3: STOPPED} and _ch(d) == [3]
    out = d.tick(M0 + 1)
    assert len(out[0]) == 0 and _ch(d) == []


@_case()
def pending_after_a_read(am, d):
    """a result a read's drain left pending belongs to the next tick, not to the one before the read; an upsert after
    the read supersedes it"""
    d.upsert([0, 1], _interval(am, 2))
    d.tick(M0)
    d.post([0, 1], [OK, FAIL])
    d.read([0, 1])
    assert _ch(d) == []
    d.upsert([1], _interval(am, 1))
    d.read([1])
    d.tick(M0 + 1)
    assert _ch(d) == [0]
    d.tick(M0 + 2)
    assert _ch(d) == []


@_case(hold="remedy")
def workflow_timeout(am, d):
    """a held run that outlives its timeout gets a Failed: listed at that tick, and the submission itself is not"""
    d.upsert([0, 1], _interval(am, 2, W=30, age=100))
    out = d.tick(M0)
    assert len(out[0]) == 2 and _ch(d) == []
    d.post([1], [OK])
    d.tick(M0 + 1)
    assert _ch(d) == [1]
    out = d.tick(M0 + 30)
    assert [i for i, _ in _timed(out)] == [0] and _ch(d) == [0]


@_case(hold="remedy")
def remedy_timeout(am, d):
    """the Failed that starts a remedy run is listed, and so is the remedy timeout's Failed"""
    d.upsert([0], _interval(am, 1, has_remedy=True, W=30, age=100))
    d.tick(M0)
    d.post([0], [FAIL])
    d.tick(M0 + 1)
    assert _ch(d) == [0]
    d.tick(M0 + 2)
    assert _ch(d) == []
    out = d.tick(M0 + 31)
    assert [int(i) for i in out[4][0]] == [0] and _ch(d) == [0]


CASES = [success_without_reset, remedy_phase_alone, superseded_result, result_on_removed_slot, anomaly, stopped_once,
         pending_after_a_read, workflow_timeout, remedy_timeout]
