"""The remedy-hold oracle (tests/remedy_hold_oracle.py) in tests/handle_model.py reproduces the hand-derived cases of
tests/remedy_hold_cases.py, and with the remedy hold off, or with no remedy action anywhere, it is the workflow-timeout
oracle's tick."""
import numpy as np
import pytest

import remedy_hold_cases
import remedy_hold_oracle
from adversarial import ZoneMap, population, zones_usable
from handle_model import NONE, HandleModel


@pytest.mark.parametrize("case", remedy_hold_cases.CASES, ids=lambda c: c.__name__)
def test_hand_derived_cases(am, orc, case):
    case(am, HandleModel(ZoneMap(), 8, hold=True, remedy=True))


def _steps(rng, n, T, zmap, st_a, st_b, remedy_actions):
    """the same random calls on two oracle states, then a tick of each; yields both results"""
    for step in [0, 1, 1, 57, 1, 2, 60, 29, 1, 3600, 1, 31]:
        if step:
            fl = np.flatnonzero(st_a.since != NONE)
            if len(fl):
                sl = rng.choice(fl, min(len(fl), 200), replace=False)
                ph = rng.integers(0, 3, len(sl)).astype(np.uint8)
                rp = rng.integers(0, 3, len(sl)).astype(np.uint8)
                for s in (st_a, st_b):
                    s.post(sl, ph, rp)
        T += step
        yield st_a.tick(T), st_b.tick(T)


@pytest.mark.parametrize("what", ["remedy_hold_off", "no_remedy_actions"])
def test_it_is_the_timeout_oracle_without_remedy_runs(am, orc, what):
    zmap = ZoneMap()
    T = 1790812800 + 13 * 86400 + 14 * 3600
    n = 4000
    rng = np.random.default_rng(11)
    cols = population(rng, n, T - 700, True, zmap.ids_of(zones_usable(T - 700, T + 2 * 86400)))
    if what == "no_remedy_actions":
        cols["flags"] &= np.uint32(~am.F_HAS_REMEDY & 0xFFFFFFFF)
    recs = am.columns_to_records(cols)
    recs["wf_timeout"] = rng.integers(0, 90, n)
    a = HandleModel(zmap, n, hold=True, remedy=True)
    if what == "remedy_hold_off":
        a.set_remedy(False)
    b = HandleModel(zmap, n, hold=True)
    a.upsert(np.arange(n), recs)
    b.upsert(np.arange(n), recs)
    seen = 0
    for ga, gb in _steps(rng, n, T, zmap, a, b, what):
        assert ga[2] == gb[2]
        np.testing.assert_array_equal(ga[0], gb[0])
        np.testing.assert_array_equal(ga[1], gb[1])
        np.testing.assert_array_equal(ga[3][0], gb[3][0])
        assert len(ga[4][0]) == 0
        np.testing.assert_array_equal(a.since, b.since)
        np.testing.assert_array_equal(a.deadline, b.deadline)
        seen += ga[2]["n_emitted"]
    for name in a.cols():
        np.testing.assert_array_equal(a.cols()[name], b.cols()[name], err_msg=name)
    assert (a.rsince == remedy_hold_oracle.NONE).all() and seen > 1000
