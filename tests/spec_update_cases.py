"""Hand-derived cases of spec updates (am_sweep_update_spec, DESIGN §6 item 20), written against a `driver`: a handle
compared with tests/spec_update_model.py after every tick (tests/test_spec_update_gpu.py, through every tick entry
point).  A driver starts with the hold, the remedy hold, status changes and their details on, and has upsert, update_spec,
remove, post, tick(T, mode=0) -> (idx, act, stats, timed_out, remedy_timed_out), in_flight() and cols()."""
import numpy as np

from timeout_cases import M0, NONE, SUBMIT, _acts, _timed, rec

OK = 1
STOPPED = 0x04
F_STOPPED_REPORTED = 1 << 9


def _echo(am, d, via):
    """RepeatAfterSec 30.  Tick 70 applies a Succeeded (S = 7, finishedAt = 70); the run submitted at 100 posts
    Succeeded at 102; the status written at 101 comes back at 103 through `via`, before tick 104 drains"""
    spec = dict(repeat_after_sec=30)
    d.upsert([0], rec(am, 0, finished_at=M0 - 100, success_count=6, **spec))
    assert _acts(d.tick(M0 + 40)) == {0: SUBMIT}
    d.post([0], [OK])
    out = d.tick(M0 + 70)
    assert out[2]["n_result_ok"] == 1 and _acts(out) == {}
    assert d.cols()["success"][0] == 7 and d.cols()["finished_at"][0] == M0 + 70
    assert _acts(d.tick(M0 + 100)) == {0: SUBMIT}
    d.post([0], [OK])
    getattr(d, via)([0], rec(am, 0, finished_at=M0 + 70, success_count=7, **spec))
    return d.tick(M0 + 104)


def echo_by_upsert_drops_the_result(am, d):
    """an upsert supersedes the result posted before it: S stays 7, finishedAt 70, and the phase's release of the hold
    makes the check due again 2 s after its run ended"""
    out = _echo(am, d, "upsert")
    assert out[2]["n_result_ok"] == 0 and _acts(out) == {0: SUBMIT}
    c = d.cols()
    assert c["success"][0] == 7 and c["finished_at"][0] == M0 + 70 and d.in_flight()[0] == M0 + 104


def echo_by_spec_update_counts_it(am, d):
    """a spec update keeps the result: S = 8, finishedAt = 104, nothing submitted before 134"""
    out = _echo(am, d, "update_spec")
    assert out[2]["n_result_ok"] == 1 and _acts(out) == {}
    c = d.cols()
    assert c["success"][0] == 8 and c["finished_at"][0] == M0 + 104 and d.in_flight()[0] == NONE
    assert _acts(d.tick(M0 + 133)) == {}
    assert _acts(d.tick(M0 + 134)) == {0: SUBMIT}


def kind_changes(am, d):
    """interval -> stopped is reported once; stopped -> stopped keeps STOPPED_REPORTED and is not reported again; a UTC
    5-field schedule -> one bound to Asia/Kolkata fires at that zone's minute; cron -> interval counts from the kept
    finishedAt, not from the finishedAt of the spec's record"""
    d.upsert([0], rec(am, 0, repeat_after_sec=600, finished_at=M0 - 10))
    d.upsert([1], rec(am, 0))
    d.upsert([2], rec(am, 0, cron="0 9 * * *"))
    d.upsert([3], rec(am, 0, cron="30 * * * *", finished_at=M0 - 30))
    assert _acts(d.tick(M0)) == {1: STOPPED}
    d.update_spec([0], rec(am, 0, finished_at=M0 + 5000))
    d.update_spec([1], rec(am, 0, has_remedy=True))
    d.update_spec([2], rec(am, 0, cron="CRON_TZ=Asia/Kolkata 31 12 * * *"))  # M0 + 60 is 12:31 in Kolkata
    d.update_spec([3], rec(am, 0, repeat_after_sec=60, finished_at=M0 + 59))
    out = d.tick(M0 + 60)
    assert _acts(out) == {0: STOPPED, 2: SUBMIT, 3: SUBMIT}, _acts(out)
    f = d.cols()["flags"]
    assert f[0] & F_STOPPED_REPORTED and f[1] & F_STOPPED_REPORTED
    assert d.cols()["finished_at"][0] == M0 + 60  # (STOPPED writes finishedAt; the spec's finishedAt is not taken)
    assert _acts(d.tick(M0 + 61)) == {}


def kind_change_while_held(am, d):
    """a held interval check turned into a 5-field one stays held past its minute; its run's phase ends the hold and
    is counted.  A held one turned into a stopped one is not submitted while the hold lasts."""
    d.upsert([0, 1], np.concatenate([rec(am, 0, repeat_after_sec=30, finished_at=M0 - 100)] * 2))
    assert _acts(d.tick(M0 + 1)) == {0: SUBMIT, 1: SUBMIT}
    d.update_spec([0], rec(am, 0, cron="* * * * *"))
    d.update_spec([1], rec(am, 0))
    out = d.tick(M0 + 60)
    assert not _acts(out).get(0, 0) & SUBMIT and d.in_flight()[0] == M0 + 1
    d.post([0, 1], [OK, OK])
    out = d.tick(M0 + 61)
    assert out[2]["n_result_ok"] == 2 and 0 not in _acts(out)
    assert _acts(d.tick(M0 + 120)).get(0) == SUBMIT


def timeout_change_during_a_run(am, d):
    """W 30 -> 100 during a run: the run times out at its own deadline (start + 30), the next run at start + 100"""
    T0 = M0 + 7
    d.upsert([0], rec(am, 30, repeat_after_sec=60, finished_at=T0 - 100))
    assert _acts(d.tick(T0)) == {0: SUBMIT}
    d.update_spec([0], rec(am, 100, repeat_after_sec=60))
    assert _timed(d.tick(T0 + 29)) == []
    assert _timed(d.tick(T0 + 30)) == [(0, T0)]
    assert _acts(d.tick(T0 + 90)) == {0: SUBMIT}
    assert _timed(d.tick(T0 + 189)) == []
    assert _timed(d.tick(T0 + 190)) == [(0, T0 + 90)]


def tombstones_are_left_alone(am, d):
    """a spec update of a never-upserted slot or of a removed one changes nothing and sweeps no further slot"""
    d.upsert([0], rec(am, 0, repeat_after_sec=60, finished_at=M0))
    d.update_spec([5], rec(am, 0, repeat_after_sec=1))
    assert len(d.tick(M0)[0]) == 0 and d.m.hwm == 1
    d.remove([0])
    d.update_spec([0], rec(am, 0, repeat_after_sec=1))
    out = d.tick(M0 + 5)
    assert len(out[0]) == 0 and d.cols()["flags"][0] == 1 << 8


CASES = [echo_by_upsert_drops_the_result, echo_by_spec_update_counts_it, kind_changes, kind_change_while_held,
         timeout_change_during_a_run, tombstones_are_left_alone]
