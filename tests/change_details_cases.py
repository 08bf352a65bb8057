"""Hand-derived cases of the change details (am_sweep_set_change_details), written against a driver: the oracle alone
(tests/handle_model.py, tests/test_change_details_oracle.py) or a handle compared with it after every tick
(tests/test_change_details_gpu.py, through every tick entry point).  A driver has upsert, remove, post, read(slots),
load(first, cols), set_details(on), tick(T, mode=0) -> (global idx, action, stats, ...), changes() and details() -> the
last tick's details (change_details_oracle.DETAIL, one per listed slot).  `hold` and `n` as in changes_cases.

Each case pins one rule of the started rule or of `applied` with values derived by hand from the reference's watch
loops (hcc.go:607-756, :788-852) and the hold's bookkeeping."""
import numpy as np

from change_details_oracle import (CHG_CLOSED_LOOP, CHG_FAILED, CHG_REMEDY_FAILED, CHG_REMEDY_SUCCEEDED,
                                   CHG_REMEDY_TIMED_OUT, CHG_STOPPED, CHG_SUCCEEDED, CHG_TIMED_OUT, NONE)
from changes_cases import _case, _interval
from timeout_cases import M0, rec

OK, FAIL, NO = 1, 2, 0
SUBMIT_HC, RUN_REMEDY, STOPPED, RESET_ON_PASS, RESET_ON_INTERVAL = 0x01, 0x02, 0x04, 0x20, 0x40
MIN = int(NONE)


def _det(d):
    """{slot: (started, remedy_started, applied, action)} of the last tick"""
    idx = np.asarray(d.changes()).tolist()
    det = d.details()
    assert len(det) == len(idx)
    return {i: (int(x["started"]), int(x["remedy_started"]), int(x["applied"]), int(x["action"])) for i, x in zip(idx, det)}


@_case(hold="hold")
def one_phase_per_run(am, d):
    """each run's phase reports the tick that submitted it"""
    d.upsert([0, 1], _interval(am, 2, age=100))
    d.tick(M0)
    d.post([0, 1], [OK, FAIL])
    d.tick(M0 + 1)
    assert _det(d) == {0: (M0, MIN, CHG_SUCCEEDED, 0), 1: (M0, MIN, CHG_FAILED, 0)}


@_case(hold="hold")
def two_phases_in_one_drain(am, d):
    """of two calls the latest phase is applied, and the first call ended the run; two entries of one call both see it"""
    d.upsert([0, 1], _interval(am, 2, age=100))
    d.tick(M0)
    d.post([0], [OK])
    d.post([0], [FAIL])
    d.post([1, 1], [OK, FAIL])
    d.tick(M0 + 1)
    assert _det(d) == {0: (MIN, MIN, CHG_FAILED, 0), 1: (M0, MIN, CHG_FAILED, 0)}


@_case(hold="hold")
def phase_after_a_read(am, d):
    """a read's drain leaves the phase pending with its start; a phase posted after the read finds no run"""
    d.upsert([0, 1], _interval(am, 2, age=100))
    d.tick(M0)
    d.post([0, 1], [FAIL, OK])
    d.read([0, 1])
    d.post([1], [FAIL])
    d.tick(M0 + 1)
    assert _det(d) == {0: (M0, MIN, CHG_FAILED, 0), 1: (MIN, MIN, CHG_FAILED, 0)}


@_case(hold="hold")
def superseded_then_posted_again(am, d):
    """an upsert drops a phase posted before it; the run that phase ended stays ended for the phase posted after"""
    d.upsert([0, 1, 2], _interval(am, 3, age=100))
    d.tick(M0)
    d.post([0, 1], [OK, OK])
    d.upsert([0, 1], _interval(am, 2, age=100))
    d.post([0], [FAIL])
    d.upsert([2], _interval(am, 1, age=100))  # (an upsert keeps the hold)
    d.post([2], [OK])
    d.tick(M0 + 1)
    assert _det(d) == {0: (MIN, MIN, CHG_FAILED, 0), 2: (M0, MIN, CHG_SUCCEEDED, 0)}


@_case(hold="hold")
def remove_upsert_phase(am, d):
    """a remove ends the run: a phase posted after the new upsert has none"""
    d.upsert([0], _interval(am, 1, age=100))
    d.tick(M0)
    d.remove([0])
    d.upsert([0], _interval(am, 1, age=100))
    d.post([0], [OK])
    d.tick(M0 + 1)
    assert _det(d) == {0: (MIN, MIN, CHG_SUCCEEDED, 0)}


@_case(hold="hold")
def load(am, d):
    """a load drops what was posted before it and ends the runs; a loaded record's own pending result has no start"""
    d.upsert([0, 1, 2], _interval(am, 3, age=100))
    d.tick(M0)
    d.post([0, 1], [OK, OK])
    recs = _interval(am, 2, age=100)
    recs["flags"][0] |= am.F_PENDING_FAIL
    d.load(1, am.records_to_columns(recs))
    d.post([2], [OK])
    d.tick(M0 + 1)
    assert _det(d) == {0: (M0, MIN, CHG_SUCCEEDED, 0), 1: (MIN, MIN, CHG_FAILED, 0), 2: (MIN, MIN, CHG_SUCCEEDED, 0)}


@_case(hold="remedy")
def timeout_with_remedy_phase_alone(am, d):
    """a workflow timeout merged with a remedy phase posted alone in the same drain: the run's start, no remedy start"""
    d.upsert([0], _interval(am, 1, has_remedy=True, W=30, age=100))
    d.tick(M0)
    d.post([0], [NO], [OK])
    d.tick(M0 + 30)
    s, rs, a, act = _det(d)[0]
    assert (s, rs, a) == (M0, MIN, CHG_FAILED | CHG_TIMED_OUT | CHG_REMEDY_SUCCEEDED) and act & RUN_REMEDY


@_case(hold="remedy", n=4)
def remedy_run_ends(am, d):
    """a remedy run ended by its remedy phase, by a workflow phase (no run of that kind: no start) and by its timeout"""
    d.upsert([0, 1, 2], _interval(am, 3, has_remedy=True, W=30, age=100))
    d.tick(M0)
    d.post([0, 1, 2], [FAIL, FAIL, FAIL])
    d.tick(M0 + 1)
    assert {i: v[:3] for i, v in _det(d).items()} == {i: (M0, MIN, CHG_FAILED) for i in range(3)}
    assert all(v[3] & RUN_REMEDY for v in _det(d).values())
    d.post([0], [NO], [OK])
    d.post([1], [OK])
    d.tick(M0 + 2)
    assert _det(d) == {0: (MIN, M0 + 1, CHG_REMEDY_SUCCEEDED, 0), 1: (MIN, MIN, CHG_SUCCEEDED, 0)}
    d.tick(M0 + 31)
    assert _det(d) == {2: (MIN, M0 + 1, CHG_REMEDY_FAILED | CHG_REMEDY_TIMED_OUT, 0)}


@_case(hold="remedy")
def attached_remedy_outcome(am, d):
    """a Failed posted with its remedy outcome: both applied, the run's start, no remedy start"""
    d.upsert([0], _interval(am, 1, has_remedy=True, age=100))
    d.tick(M0)
    d.post([0], [FAIL], [OK])
    d.tick(M0 + 1)
    s, rs, a, act = _det(d)[0]
    assert (s, rs, a) == (M0, MIN, CHG_FAILED | CHG_REMEDY_SUCCEEDED) and act & RUN_REMEDY


@_case()
def resets(am, d):
    """the reset on a pass and on an elapsed interval are read from the action"""
    d.upsert([0], rec(am, 0, repeat_after_sec=60, finished_at=M0 - 10, has_remedy=True, remedy_total_runs=1))
    d.upsert([1], rec(am, 0, repeat_after_sec=60, finished_at=M0 - 10, has_remedy=True, remedy_runs_limit=1,
                      remedy_reset_interval=60, remedy_total_runs=1, remedy_finished_at=M0 - 1000))
    d.post([0, 1], [OK, FAIL])
    d.tick(M0)
    got = _det(d)
    assert got[0] == (MIN, MIN, CHG_SUCCEEDED, RESET_ON_PASS)
    assert got[1][:3] == (MIN, MIN, CHG_FAILED) and got[1][3] & RESET_ON_INTERVAL and got[1][3] & RUN_REMEDY


@_case()
def anomaly_is_not_listed(am, d):
    d.upsert([0, 1], np.concatenate([rec(am, 0, repeat_after_sec=60, finished_at=M0 - 10, has_remedy=True,
                                         remedy_runs_limit=1, remedy_reset_interval=60, remedy_total_runs=1)] * 2))
    d.post([0, 1], [FAIL, OK])
    d.tick(M0)
    assert _det(d) == {1: (MIN, MIN, CHG_SUCCEEDED, RESET_ON_PASS)}


@_case()
def stopped(am, d):
    d.upsert([3], rec(am, 0, repeat_after_sec=0))
    d.upsert([4], rec(am, 0, repeat_after_sec=0))
    d.post([4], [FAIL])
    d.tick(M0)
    assert _det(d) == {3: (MIN, MIN, CHG_STOPPED, STOPPED), 4: (MIN, MIN, CHG_STOPPED | CHG_FAILED, STOPPED)}


@_case()
def closed_loop(am, d):
    """a record due in a closed-loop tick completes in it: started = T"""
    d.upsert([0, 1], _interval(am, 2, age=100))
    d.upsert([2], _interval(am, 1, age=10))
    d.post([2], [OK])
    d.tick(M0, 0x1)
    got = _det(d)
    assert got[0] == got[1] == (M0, MIN, CHG_CLOSED_LOOP, SUBMIT_HC) and got[2] == (MIN, MIN, CHG_SUCCEEDED, 0)


@_case()
def hold_off(am, d):
    """with the hold off the library sees no run start"""
    d.upsert([0], _interval(am, 1, age=100))
    d.tick(M0)
    d.post([0], [FAIL])
    d.tick(M0 + 1)
    assert _det(d) == {0: (MIN, MIN, CHG_FAILED, 0)}


@_case(hold="hold")
def pending_from_before_details(am, d):
    """a phase posted while details are off has no start, nor has a tick's list from before they were turned on"""
    d.upsert([0, 1], _interval(am, 2, age=100))
    d.tick(M0)
    d.set_details(False)
    d.post([0], [OK])
    d.tick(M0 + 1)
    d.post([1], [OK])
    d.set_details(True)
    assert len(d.details()) == 0
    d.tick(M0 + 2)
    assert _det(d) == {1: (MIN, MIN, CHG_SUCCEEDED, 0)}


CASES = [one_phase_per_run, two_phases_in_one_drain, phase_after_a_read, superseded_then_posted_again,
         remove_upsert_phase, load, timeout_with_remedy_phase_alone, remedy_run_ends, attached_remedy_outcome, resets,
         anomaly_is_not_listed, stopped, closed_loop, hold_off, pending_from_before_details]
