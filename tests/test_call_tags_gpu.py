"""The entries of one post call see the in-flight state from before the call, and only they do: the change details tell
two post calls of one drain apart exactly.  Each staged result op carries its call's first op index mod 2^22, so the
cases put the second call's first op exactly 2^22 ops after the first call's (equal tags), one op short of that (the
control: the tags differ), and both entries of the slot into one call of more than 2^22 entries.  The details of the
tick that applies them are compared with tests/handle_model.py through tests/handle_pair.py."""
import numpy as np
import pytest

from adversarial import ZoneMap
from change_details_oracle import NONE
from changes_cases import _interval
from handle_pair import Pair
from timeout_cases import M0

pytestmark = pytest.mark.gpu

TAG = 1 << 22  # the op index span of a call tag
OK, FAIL, NO = 1, 2, 0
GAPS = {"apart_2_22": TAG, "apart_2_22_less_1": TAG - 1, "one_call_over_2_22": TAG + 5}


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


def _calls(layout, run):
    """[(slots, phases, remedy phases)] of the post calls: slot 0's first phase, filler entries without a phase on
    slot 1 up to `gap`, slot 0's second phase; split into three calls, or one call for "one_call_over_2_22".  `run`
    "hold" posts workflow phases (Succeeded, then Failed), "remedy" remedy phases."""
    gap = GAPS[layout]
    slots = np.ones(gap + 1, np.uint64)
    slots[[0, -1]] = 0
    ph, rph = np.zeros(gap + 1, np.uint8), np.zeros(gap + 1, np.uint8)
    (ph if run == "hold" else rph)[[0, -1]] = OK, FAIL
    if layout == "one_call_over_2_22":
        return [(slots, ph, rph)]
    return list(zip(*(np.split(a, [1, gap]) for a in (slots, ph, rph))))


@pytest.mark.parametrize("layout", list(GAPS))
@pytest.mark.parametrize("run", ["hold", "remedy"])
def test_a_call_sees_the_runs_its_drain_ended_before_it(am, zmap, run, layout):
    p = Pair(am, zmap, 8, hold=True, remedy=run == "remedy", track=True, details=True, every_slot=False)
    try:
        p.upsert([0, 1], _interval(am, 2, has_remedy=True, age=100))
        p.tick(M0)
        T, start = M0 + 1, M0
        if run == "remedy":  # a Failed starts the remedy run at the tick that applies it
            p.post([0], [FAIL])
            p.tick(T)
            T, start = T + 1, M0 + 1
            assert p.m.remedy_in_flight(idx=[0])[0] == start
        else:
            assert p.m.in_flight(idx=[0])[0] == start
        calls = _calls(layout, run)
        for slots, ph, rph in calls:
            p.post(slots, ph, rph)
        p.tick(T)  # (compares the details with the model's)
        det = dict(zip(p.m.changes().tolist(), p.m.details()))
        got = int(det[0]["remedy_started" if run == "remedy" else "started"])
        # two calls: the first ended the run, so the second sees nothing in flight; one call: every entry sees the run
        assert got == (start if len(calls) == 1 else int(NONE)), (layout, got)
        assert sum(len(c[0]) for c in calls) == GAPS[layout] + 1
    finally:
        p.close()
