"""The workflow-timeout oracle (tests/timeout_oracle.py) in tests/handle_model.py reproduces the hand-derived cases of
tests/timeout_cases.py, and with no deadline anywhere it is the hold oracle's tick."""
import numpy as np
import pytest

import hold_oracle
import timeout_cases
import timeout_oracle
from adversarial import ZoneMap, population, zones_usable
from handle_model import HandleModel


@pytest.mark.parametrize("case", timeout_cases.CASES, ids=lambda c: c.__name__)
def test_hand_derived_cases(am, orc, case):
    case(am, HandleModel(ZoneMap(), 8, hold=True))


def test_without_deadlines_it_is_the_hold_oracle(am, orc):
    zmap = ZoneMap()
    T = 1790812800 + 13 * 86400 + 14 * 3600
    n = 5000
    rng = np.random.default_rng(5)
    cols = population(rng, n, T - 700, True, zmap.ids_of(zones_usable(T - 700, T)))
    a = {k: v.copy() for k, v in cols.items()}
    b = {k: v.copy() for k, v in cols.items()}
    sa, sb = hold_oracle.none_in_flight(n), hold_oracle.none_in_flight(n)
    d = timeout_oracle.no_deadlines(n)
    wf = np.zeros(n, dtype=np.int32)
    for t in (T, T + 1, T + 60, T + 3600):
        gi, ga, gs, timed = timeout_oracle.sweep(zmap, a, sa, d, wf, t)
        wi, wa, ws = hold_oracle.sweep(zmap, b, sb, t)
        assert gs == ws and len(timed[0]) == 0
        np.testing.assert_array_equal(gi, wi)
        np.testing.assert_array_equal(ga, wa)
        np.testing.assert_array_equal(sa, sb)
    assert (d == timeout_oracle.NO_DEADLINE).all()
