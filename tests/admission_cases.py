"""Hand-derived cases of the submit budget (am_sweep_set_submit_budget, DESIGN §6 item 19), written against a `driver`:
the model alone (tests/admission_model.py) or a handle compared with it after every tick (tests/test_admission_gpu.py,
through every tick entry point).  A driver starts with the hold and the remedy hold on and has upsert, remove, load,
post, tick(T, mode=0) -> (idx, act, stats, timed_out, remedy_timed_out), set_budget(per_tick), deferred(),
in_flight(), remedy_in_flight() and last_admission()."""
import numpy as np

import admission_oracle as ao
from timeout_cases import M0, NONE, RUN_REMEDY, SUBMIT, _acts, _timed, rec

FAIL = 2
CATCH_UP = 0x8
W = ao.NOT_WAITING


def _adm(d, n_candidates, n_admitted, n_deferred, oldest):
    assert d.last_admission() == {"n_candidates": n_candidates, "n_admitted": n_admitted, "n_deferred": n_deferred,
                                  "oldest_deferred": oldest}, d.last_admission()


def budget_zero(am, d):
    """budget 0: nothing is submitted and every candidate waits from T; then the oldest go first, by index"""
    d.upsert([0, 1, 2], np.concatenate([rec(am, 0, repeat_after_sec=60, finished_at=M0 - 100)] * 3))
    d.set_budget(0)
    out = d.tick(M0 + 5)
    assert _acts(out) == {} and out[2]["n_submit_hc"] == 0 and out[2]["n_emitted"] == 0
    assert d.deferred()[:3].tolist() == [M0 + 5] * 3 and d.in_flight()[:3].tolist() == [NONE] * 3
    _adm(d, 3, 0, 3, M0 + 5)
    d.set_budget(2)
    out = d.tick(M0 + 6)
    assert _acts(out) == {0: SUBMIT, 1: SUBMIT}
    assert d.in_flight()[:3].tolist() == [M0 + 6, M0 + 6, NONE] and d.deferred()[:3].tolist() == [W, W, M0 + 5]
    _adm(d, 3, 2, 1, M0 + 5)


def cron_across_two_activations(am, d):
    """a 5-field check that waits across two of its minutes is submitted once, at the tick that admits it"""
    d.upsert([0], rec(am, 0, cron="* * * * *"))
    d.set_budget(0)
    assert _acts(d.tick(M0)) == {}
    assert _acts(d.tick(M0 + 60)) == {}
    assert d.deferred()[0] == M0  # (the first second it waited)
    d.set_budget(1)
    out = d.tick(M0 + 61)  # off the minute: due only because it waits
    assert _acts(out) == {0: SUBMIT} and d.in_flight()[0] == M0 + 61 and d.deferred()[0] == W
    assert _acts(d.tick(M0 + 62)) == {}


def waits_end(am, d):
    """an upsert keeps the wait; a remove, a load and a posted workflow phase end it"""
    d.upsert([0, 1, 2, 3], np.concatenate([rec(am, 0, repeat_after_sec=60, finished_at=M0 - 100)] * 4))
    d.set_budget(0)
    d.tick(M0 + 1)
    assert d.deferred()[:4].tolist() == [M0 + 1] * 4
    d.upsert([0], rec(am, 0, repeat_after_sec=600, finished_at=M0))  # not due by its rule any more: still waiting
    d.remove([1])
    cols = {k: v[2:3].copy() for k, v in d.cols().items()}
    d.load(2, cols)
    d.post([3], [FAIL])
    assert d.deferred()[:4].tolist() == [M0 + 1, W, W, W]
    d.set_budget(None)
    out = d.tick(M0 + 2)
    assert _acts(out).get(0) == SUBMIT and 1 not in _acts(out)  # the upserted one is admitted all the same


def remedy_run_on_a_waiting_check(am, d):
    """a Failed posted for a waiting check ends its wait; the tick runs its remedy, holds it and does not submit it"""
    d.upsert([0], rec(am, 0, repeat_after_sec=60, finished_at=M0 - 100, has_remedy=True, remedy_runs_limit=3))
    d.set_budget(0)
    d.tick(M0 + 1)
    d.post([0], [FAIL])
    out = d.tick(M0 + 2)
    assert _acts(out) == {0: RUN_REMEDY} and d.remedy_in_flight()[0] == M0 + 2 and d.deferred()[0] == W


def timeout_from_admission(am, d):
    """W = 30: a check that waited from M0 + 1 and was admitted at M0 + 40 times out at M0 + 70, StartedAt M0 + 40"""
    d.upsert([0], rec(am, 30, repeat_after_sec=60, finished_at=M0 - 100))
    d.set_budget(0)
    for t in (1, 14, 27):
        out = d.tick(M0 + t)
        assert _acts(out) == {} and _timed(out) == []
    d.set_budget(1)
    assert _acts(d.tick(M0 + 40)) == {0: SUBMIT}
    assert _timed(d.tick(M0 + 69)) == []
    assert _timed(d.tick(M0 + 70)) == [(0, M0 + 40)]


def catch_up_window(am, d):
    """a waiting 5-field check and a catch-up tick whose window holds two more activations: submitted once"""
    d.upsert([0, 1], np.concatenate([rec(am, 0, cron="* * * * *")] * 2))
    d.set_budget(1)
    assert _acts(d.tick(M0)) == {0: SUBMIT}  # slot 1 waits
    d.post([0], [1])
    out = d.tick(M0 + 150, CATCH_UP)  # (M0, M0 + 150] holds M0 + 60 and M0 + 120: both fire, slot 1 goes first
    assert _acts(out) == {1: SUBMIT} and d.deferred()[:2].tolist() == [M0 + 150, W]


CASES = [budget_zero, cron_across_two_activations, waits_end, remedy_run_on_a_waiting_check, timeout_from_admission,
         catch_up_window]
