"""Hand-derived cases of the remedy hold (am_sweep_set_hold_remedy, with the hold in flight on), written against a
`driver`: the model alone (tests/handle_model.py) or a handle compared with it after every tick
(tests/test_remedy_hold_gpu.py, through every tick entry point).  A driver starts with the hold and the remedy hold on
and has upsert(slots, recs), remove(slots), load(first, cols), post(slots, phase, rphase=None), tick(T, mode=0) ->
(global idx, action, stats, (timed-out idx, since), (remedy timed-out idx, start)), in_flight(), remedy_in_flight(),
cols(), set_hold(on) and set_remedy(on), which raise handle_model.Refused when refused."""
import numpy as np

from handle_model import Refused
from timeout_cases import M0, NONE, REMEDY_SKIP, RUN_REMEDY, SUBMIT, _acts, _timed, rec

OK, FAIL = 1, 2


def _rc(call, on):
    """the return code of a switch: 0, or the code it was refused with"""
    try:
        call(on)
    except Refused as r:
        return r.code
    return 0


def _rtimed(out):
    return list(zip(np.asarray(out[4][0]).tolist(), np.asarray(out[4][1]).tolist()))


def _quiet(d, ts):
    for t in ts:
        out = d.tick(t)
        assert len(out[0]) == 0 and _timed(out) == [] and _rtimed(out) == [], (t, _acts(out))


def _slow_remedies(am, d):
    """a 30-s check whose runs fail 5 s after they start and whose remedies take 300 s, ticked every 5 s for 900 s:
    (remedies started, remedy skips, most remedies running at once)"""
    T0 = M0 + 3
    d.upsert([0], rec(am, 0, repeat_after_sec=30, finished_at=T0 - 100, has_remedy=True, remedy_runs_limit=2,
                      remedy_reset_interval=300))
    fail_at, remedy_end, started, skips, most = [], [], 0, 0, 0
    for t in range(T0, T0 + 900, 5):
        ends = [e for e in remedy_end if e <= t]
        remedy_end = [e for e in remedy_end if e > t]
        if t in fail_at or ends:
            d.post([0], [FAIL if t in fail_at else am.PHASE_NONE], [FAIL if ends else am.PHASE_NONE])
        a = _acts(d.tick(t)).get(0, 0)
        if a & SUBMIT:
            fail_at.append(t + 5)
        if a & RUN_REMEDY:
            started += 1
            remedy_end.append(t + 300)
        skips += (a & REMEDY_SKIP) != 0
        most = max(most, len(remedy_end))
    return started, skips, most


def slow_remedy_limit(am, d):
    """one remedy per failure and none while it runs: two remedies, then REMEDY_SKIP (limit 2 within 300 s)"""
    started, skips, most = _slow_remedies(am, d)
    assert started == 2 and skips >= 1 and most == 1, (started, skips, most)


def slow_remedy_without_the_hold(am, d):
    """the same sequence without the remedy hold: every failure while a remedy runs reads RemedyTotalRuns == 0 and
    starts another (the defect the remedy hold removes)"""
    assert _rc(d.set_remedy, False) == 0
    started, skips, most = _slow_remedies(am, d)
    assert started > 2 and most > 2, (started, skips, most)


def merged_remedy_holds_nothing(am, d):
    """a remedy phase applied with the Failed (the same call, or two calls before one tick): nothing is held, and a
    5-field check matching the tick is submitted in it"""
    d.upsert([0, 1], np.concatenate([rec(am, 0, cron="* * * * *", has_remedy=True)] * 2))
    assert _acts(d.tick(M0)) == {0: SUBMIT, 1: SUBMIT}
    d.post([0], [FAIL], [OK])
    d.post([1], [am.PHASE_NONE], [OK])
    d.post([1], [FAIL])
    out = d.tick(M0 + 60)
    assert _acts(out) == {0: SUBMIT | RUN_REMEDY, 1: SUBMIT | RUN_REMEDY}
    assert out[2]["n_remedy_ok"] == 2 and out[2]["n_submit_hc"] == 2
    assert (d.remedy_in_flight()[:2] == NONE).all()


def cron_not_submitted_when_remedy_starts(am, d):
    """a 5-field check matching T at the tick its Failed is applied runs its remedy and is not submitted; it is
    submitted at the first matching tick after the remedy phase"""
    d.upsert([0], rec(am, 0, cron="* * * * *", has_remedy=True))
    assert _acts(d.tick(M0)) == {0: SUBMIT}
    d.post([0], [FAIL])
    out = d.tick(M0 + 60)
    assert _acts(out) == {0: RUN_REMEDY} and out[2]["n_submit_hc"] == 0
    assert d.remedy_in_flight()[0] == M0 + 60 and d.in_flight()[0] == NONE
    _quiet(d, [M0 + 120, M0 + 180])
    d.post([0], [am.PHASE_NONE], [OK])
    out = d.tick(M0 + 190)
    assert len(out[0]) == 0 and out[2]["n_remedy_ok"] == 1
    assert d.remedy_in_flight()[0] == NONE
    assert _acts(d.tick(M0 + 240)) == {0: SUBMIT}


def due_at_release(am, d):
    """a remedy phase releases the check: submitted at that tick when finishedAt + RepeatAfterSec has passed"""
    T0 = M0 + 7
    d.upsert([0, 1], np.concatenate([rec(am, 0, repeat_after_sec=60, finished_at=T0 - 100, has_remedy=True),
                                     rec(am, 0, repeat_after_sec=600, finished_at=T0 - 1000, has_remedy=True)]))
    assert _acts(d.tick(T0)) == {0: SUBMIT, 1: SUBMIT}
    d.post([0, 1], [FAIL, FAIL])
    assert _acts(d.tick(T0 + 10)) == {0: RUN_REMEDY, 1: RUN_REMEDY}
    _quiet(d, [T0 + 70, T0 + 100])
    d.post([0, 1], [am.PHASE_NONE] * 2, [OK, FAIL])
    out = d.tick(T0 + 101)
    assert _acts(out) == {0: SUBMIT} and out[2]["n_remedy_ok"] == 1 and out[2]["n_remedy_fail"] == 1
    _quiet(d, [T0 + 609])
    assert _acts(d.tick(T0 + 610)) == {1: SUBMIT}


def remedy_times_out(am, d):
    """W = 30: the remedy started at T0 + 10 times out at T0 + 40 as a posted remedy Failed; the health-check deadline
    of the run before it does not fire"""
    T0 = M0 + 13
    d.upsert([0], rec(am, 30, repeat_after_sec=600, finished_at=T0 - 1000, has_remedy=True))
    assert _acts(d.tick(T0)) == {0: SUBMIT}
    d.post([0], [FAIL])
    assert _acts(d.tick(T0 + 10)) == {0: RUN_REMEDY}
    _quiet(d, [T0 + 30, T0 + 39])
    out = d.tick(T0 + 40)
    assert len(out[0]) == 0 and _rtimed(out) == [(0, T0 + 10)] and _timed(out) == []
    assert out[2]["n_remedy_fail"] == 1
    c = d.cols()
    assert c["remedy_failed"][0] == 1 and c["remedy_total"][0] == 1 and c["remedy_finished_at"][0] == T0 + 40
    assert d.remedy_in_flight()[0] == NONE
    _quiet(d, [T0 + 609])
    assert _acts(d.tick(T0 + 610)) == {0: SUBMIT}


def workflow_timeout_starts_remedy(am, d):
    """a workflow timeout's synthetic Failed runs the remedy, which is held and times out in its turn"""
    T0 = M0 + 17
    d.upsert([0], rec(am, 30, repeat_after_sec=600, finished_at=T0 - 1000, has_remedy=True))
    assert _acts(d.tick(T0)) == {0: SUBMIT}
    out = d.tick(T0 + 30)
    assert _acts(out) == {0: RUN_REMEDY} and _timed(out) == [(0, T0)] and _rtimed(out) == []
    assert d.remedy_in_flight()[0] == T0 + 30 and d.in_flight()[0] == NONE
    _quiet(d, [T0 + 59])
    out = d.tick(T0 + 60)
    assert _rtimed(out) == [(0, T0 + 30)] and out[2]["n_remedy_fail"] == 1 and len(out[0]) == 0


def releases(am, d):
    """a stray workflow phase, a remove, a load and the remedy hold turned off end a remedy run; an upsert does not;
    turning the hold off and on ends them as well and leaves the remedy hold off"""
    r = rec(am, 0, cron="* * * * *", has_remedy=True)
    d.upsert(np.arange(5), np.concatenate([r] * 5))
    assert len(d.tick(M0)[0]) == 5
    d.post(np.arange(5), [FAIL] * 5)
    assert _acts(d.tick(M0 + 60)) == {k: RUN_REMEDY for k in range(5)}
    d.post([0], [OK])
    d.remove([1])
    d.load(2, am.records_to_columns(r))
    d.upsert([3], r)
    out = d.tick(M0 + 61)
    assert out[2]["n_result_ok"] == 1 and len(out[0]) == 0
    assert d.remedy_in_flight()[:5].tolist() == [NONE, NONE, NONE, M0 + 60, M0 + 60]
    assert _rc(d.set_remedy, False) == 0 and _rc(d.set_remedy, True) == 0
    assert (d.remedy_in_flight() == NONE).all()
    d.post([3], [FAIL])
    out = d.tick(M0 + 120)
    assert _acts(out) == {0: SUBMIT, 2: SUBMIT, 3: RUN_REMEDY, 4: SUBMIT}
    assert d.remedy_in_flight()[3] == M0 + 120
    assert _rc(d.set_hold, False) == 0 and _rc(d.set_hold, True) == 0
    assert (d.remedy_in_flight() == NONE).all() and (d.in_flight() == NONE).all()
    d.post([4], [FAIL])
    assert _acts(d.tick(M0 + 180)) == {k: SUBMIT for k in (0, 2, 3)} | {4: SUBMIT | RUN_REMEDY}


def refused_without_the_hold(am, d):
    """am_sweep_set_hold_remedy while the hold in flight is off returns AM_E_INVAL and changes nothing"""
    assert _rc(d.set_hold, False) == 0
    assert _rc(d.set_remedy, True) == am.AM_E_INVAL and _rc(d.set_remedy, False) == am.AM_E_INVAL
    assert _rc(d.set_hold, True) == 0
    d.upsert([0], rec(am, 0, cron="* * * * *", has_remedy=True))
    assert _acts(d.tick(M0)) == {0: SUBMIT}
    d.post([0], [FAIL])
    assert _acts(d.tick(M0 + 60)) == {0: SUBMIT | RUN_REMEDY}  # the remedy hold stayed off
    assert _rc(d.set_remedy, True) == 0


CASES = [slow_remedy_limit, slow_remedy_without_the_hold, merged_remedy_holds_nothing,
         cron_not_submitted_when_remedy_starts, due_at_release, remedy_times_out, workflow_timeout_starts_remedy,
         releases, refused_without_the_hold]
