"""The submit-budget model (tests/admission_model.py) reproduces the hand-derived cases of tests/admission_cases.py, and
with no budget ever set it is the model it extends."""
import numpy as np
import pytest

import admission_cases
from adversarial import ZoneMap, population, zones_usable
from admission_model import AdmissionModel
from handle_model import NONE, HandleModel


@pytest.mark.parametrize("case", admission_cases.CASES, ids=lambda c: c.__name__)
def test_hand_derived_cases(am, orc, case):
    case(am, AdmissionModel(ZoneMap(), 8, hold=True, remedy=True))


def test_an_unlimited_budget_is_the_handle_model(am, orc):
    """a finite budget set and made unlimited again before any tick: every tick is the model's own"""
    zmap = ZoneMap()
    T = 1790812800 + 13 * 86400 + 14 * 3600
    n = 3000
    rng = np.random.default_rng(4)
    cols = population(rng, n, T - 700, True, zmap.ids_of(zones_usable(T - 700, T + 2 * 86400)))
    a, b = HandleModel(zmap, n, hold=True, remedy=True), AdmissionModel(zmap, n, hold=True, remedy=True)
    b.set_budget(5)
    b.set_budget(None)
    for m in (a, b):
        m.load(0, {k: v.copy() for k, v in cols.items()})
    for step in [0, 1, 59, 1, 60, 2]:
        T += step
        fl = np.flatnonzero(a.since != NONE)
        sl = rng.choice(fl, min(len(fl), 100), replace=False) if len(fl) else fl
        ph = rng.integers(1, 3, len(sl)).astype(np.uint8)
        for m in (a, b):
            m.post(sl, ph)
        x, y = a.tick(T), b.tick(T)
        np.testing.assert_array_equal(x.idx, y.idx)
        np.testing.assert_array_equal(x.act, y.act)
        assert x.stats == y.stats
    assert b.last_admission()["n_deferred"] == 0 and b.last_admission()["n_admitted"] > 0
