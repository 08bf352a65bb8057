"""Hand-derived cases of workflow timeouts (am_record_t.wf_timeout with the hold in flight on), written against a
`driver`: the model alone (tests/handle_model.py) or a handle compared with it after every tick
(tests/test_workflow_timeout_gpu.py, through every tick entry point).  A driver has upsert(slots, recs),
post(slots, phase, rphase=None), tick(T, mode=0) -> (global idx, action, stats, (timed-out idx, since)),
in_flight() -> since per slot, and cols() -> the sixteen columns."""
import numpy as np

NONE = -(1 << 63)
SUBMIT, RUN_REMEDY, REMEDY_SKIP = 0x01, 0x02, 0x10
CATCH_UP = 0x8
M0 = 1790812800 + 3 * 86400 + 7 * 3600  # on a UTC minute


def rec(am, W, **kw):
    rc, r = am.classify(**kw)
    assert rc == 0
    r["wf_timeout"] = W
    return r


def _acts(out):
    return dict(zip(np.asarray(out[0]).tolist(), np.asarray(out[1]).tolist()))


def _timed(out):
    return list(zip(np.asarray(out[3][0]).tolist(), np.asarray(out[3][1]).tolist()))


def _quiet(d, ts):
    for t in ts:
        out = d.tick(t)
        assert len(out[0]) == 0 and _timed(out) == [], (t, _acts(out), _timed(out))


def interval_expires(am, d):
    """W = 30, no phase posted: held until T0 + 29; at T0 + 30 Failed + 1, finishedAt = T0 + 30, no submission; the
    timer submits it again at T0 + 30 + RepeatAfterSec"""
    T0 = M0 + 7
    d.upsert([0], rec(am, 30, repeat_after_sec=60, finished_at=T0 - 100))
    assert _acts(d.tick(T0)) == {0: SUBMIT}
    _quiet(d, range(T0 + 1, T0 + 30))
    assert d.in_flight()[0] == T0
    out = d.tick(T0 + 30)
    assert len(out[0]) == 0 and _timed(out) == [(0, T0)] and out[2]["n_result_fail"] == 1
    c = d.cols()
    assert c["failed"][0] == 1 and c["finished_at"][0] == T0 + 30
    assert d.in_flight()[0] == NONE
    _quiet(d, range(T0 + 31, T0 + 90))
    assert _acts(d.tick(T0 + 90)) == {0: SUBMIT}
    assert d.in_flight()[0] == T0 + 90


def phase_wins(am, d):
    """a phase posted before the deadline tick wins: in an earlier drain, or in the deadline tick's own"""
    T0 = M0 + 11
    d.upsert([0, 1], np.concatenate([rec(am, 30, repeat_after_sec=600, finished_at=T0 - 1000)] * 2))
    assert _acts(d.tick(T0)) == {0: SUBMIT, 1: SUBMIT}
    d.post([0], [am.PHASE_SUCCEEDED])
    out = d.tick(T0 + 10)
    assert out[2]["n_result_ok"] == 1 and _timed(out) == []
    d.post([1], [am.PHASE_SUCCEEDED])
    out = d.tick(T0 + 30)
    assert out[2]["n_result_ok"] == 1 and out[2]["n_result_fail"] == 0 and _timed(out) == []
    c = d.cols()
    assert c["success"][0] == 1 and c["success"][1] == 1 and c["failed"][0] == 0 and c["failed"][1] == 0


def remedy_at_expiry(am, d):
    """a remedy check runs its remedy (or skips it) at expiry, as after a posted Failed.  Slot 2 and 3 also have a
    remedy phase posted alone in the expiry tick's drain: it is applied together with the synthetic Failed (the gate
    sees the remedy state before it), as behind a Failed posted after it"""
    T0 = M0 + 13
    base = dict(repeat_after_sec=600, finished_at=T0 - 1000, has_remedy=True)
    recs = [rec(am, 30, **base),  # no limit: RUN_REMEDY
            rec(am, 30, remedy_runs_limit=1, remedy_reset_interval=3600, remedy_total_runs=1,
                remedy_finished_at=T0 - 10, **base),  # limit reached within the reset interval: REMEDY_SKIP
            rec(am, 30, **base),  # no limit, remedy phase alone in the same drain
            rec(am, 30, remedy_runs_limit=1, remedy_reset_interval=3600, **base)]  # one run left, remedy phase alone
    d.upsert([0, 1, 2, 3], np.concatenate(recs))
    assert set(_acts(d.tick(T0)).values()) == {SUBMIT}
    d.post([2, 3], [am.PHASE_NONE] * 2, [am.PHASE_SUCCEEDED] * 2)
    out = d.tick(T0 + 30)
    a = _acts(out)
    assert a[0] & RUN_REMEDY and a[1] & REMEDY_SKIP and a[2] & RUN_REMEDY and a[3] & RUN_REMEDY, a
    assert _timed(out) == [(0, T0), (1, T0), (2, T0), (3, T0)]
    assert out[2]["n_result_fail"] == 4 and out[2]["n_remedy_ok"] == 2


def cron_expiry(am, d):
    """an every-minute check with W = 90 expires off the minute and is submitted at the next minute; one with W = 120
    expires on a minute that matches, and is submitted again in the same tick"""
    d.upsert([0, 1], np.concatenate([rec(am, 90, cron="* * * * *"), rec(am, 120, cron="* * * * *")]))
    assert _acts(d.tick(M0)) == {0: SUBMIT, 1: SUBMIT}
    out = d.tick(M0 + 60)
    assert len(out[0]) == 0 and _timed(out) == []
    out = d.tick(M0 + 90)
    assert len(out[0]) == 0 and _timed(out) == [(0, M0)] and out[2]["n_result_fail"] == 1
    out = d.tick(M0 + 120)
    assert _acts(out) == {0: SUBMIT, 1: SUBMIT} and _timed(out) == [(1, M0)]
    f = d.in_flight()
    assert f[0] == M0 + 120 and f[1] == M0 + 120
    c = d.cols()
    assert c["failed"][0] == 1 and c["failed"][1] == 1 and c["finished_at"][1] == M0 + 120


def skipped_seconds(am, d):
    """ticks at T0 and T0 + 150 only: both runs time out at the late tick; with AM_SWEEP_CATCH_UP the every-minute
    check is due by its window and submitted again in the same tick"""
    d.upsert([0, 1], np.concatenate([rec(am, 30, repeat_after_sec=60, finished_at=M0 - 100),
                                     rec(am, 30, cron="* * * * *")]))
    assert _acts(d.tick(M0)) == {0: SUBMIT, 1: SUBMIT}
    out = d.tick(M0 + 150, mode=CATCH_UP)
    assert _acts(out) == {1: SUBMIT} and _timed(out) == [(0, M0), (1, M0)]
    c = d.cols()
    assert c["finished_at"][0] == M0 + 150 and c["failed"][0] == 1
    assert d.in_flight()[1] == M0 + 150


def upsert_mid_run(am, d):
    """an upsert during a run changes the timeout of the next run only"""
    T0 = M0 + 17
    d.upsert([0], rec(am, 30, repeat_after_sec=60, finished_at=T0 - 100))
    assert _acts(d.tick(T0)) == {0: SUBMIT}
    d.upsert([0], rec(am, 100, repeat_after_sec=60, finished_at=T0 - 100))  # still held: finishedAt <= since
    _quiet(d, [T0 + 5, T0 + 29])
    assert _timed(d.tick(T0 + 30)) == [(0, T0)]
    assert _acts(d.tick(T0 + 90)) == {0: SUBMIT}
    _quiet(d, [T0 + 120, T0 + 189])
    assert _timed(d.tick(T0 + 190)) == [(0, T0 + 90)]


def released_then_held(am, d):
    """a run released by an upsert with a later finishedAt is not timed out, and an upsert that holds it again after
    its deadline tick does not bring the deadline back"""
    T0 = M0 + 19
    d.upsert([0], rec(am, 30, repeat_after_sec=3600, finished_at=T0 - 5000))
    assert _acts(d.tick(T0)) == {0: SUBMIT}
    d.upsert([0], rec(am, 30, repeat_after_sec=3600, finished_at=T0 + 10))
    _quiet(d, [T0 + 10, T0 + 30])
    d.upsert([0], rec(am, 30, repeat_after_sec=3600, finished_at=T0 - 100))
    assert d.in_flight()[0] == T0
    _quiet(d, [T0 + 31, T0 + 1000, T0 + 3500, T0 + 3600])
    assert d.in_flight()[0] == T0 and d.cols()["failed"][0] == 0


def zero_never_expires(am, d):
    """W = 0: no deadline, the run stays held"""
    T0 = M0 + 23
    d.upsert([0], rec(am, 0, repeat_after_sec=60, finished_at=T0 - 100))
    assert _acts(d.tick(T0)) == {0: SUBMIT}
    _quiet(d, [T0 + 30, T0 + 1000, T0 + 86400])
    assert d.in_flight()[0] == T0


CASES = [interval_expires, phase_wins, remedy_at_expiry, cron_expiry, skipped_seconds, upsert_mid_run,
         released_then_held, zero_never_expires]
