"""The remedy-hold oracle (tests/remedy_hold_oracle.py) reproduces the hand-derived cases of tests/remedy_hold_cases.py,
and with the remedy hold off, or with no remedy action anywhere, it is the workflow-timeout oracle's tick."""
import numpy as np
import pytest

import remedy_hold_cases
import remedy_hold_oracle
import timeout_oracle
from adversarial import ZoneMap, population, zones_usable


class OracleDriver:
    """the oracle side alone, with the switches a handle has (the oracle's State assumes the hold is on)"""

    def __init__(self, am, n=8):
        self.am = am
        self.st = remedy_hold_oracle.State(ZoneMap(), am.records_to_columns(np.zeros(n, dtype=am.RECORD_DTYPE)))
        self.st.ocols["flags"][:] = am.F_TOMBSTONE
        self.hold = True

    def upsert(self, slots, recs):
        self.st.upsert(slots, recs)

    def remove(self, slots):
        self.st.remove(slots)

    def load(self, first, cols):
        self.st.load(first, cols)

    def post(self, slots, phase, rphase=None):
        self.st.post(slots, phase, rphase)

    def tick(self, T, mode=0):
        return self.st.tick(T, mode)

    def in_flight(self):
        return self.st.in_flight()

    def remedy_in_flight(self):
        return self.st.remedy_in_flight()

    def cols(self):
        return self.st.ocols

    def set_hold(self, on):
        if self.hold and not on:
            self.st.hold_on_again()  # (the state a handle has when the hold is turned on again)
        self.hold = bool(on)
        return 0

    def set_remedy(self, on):
        if not self.hold:
            return self.am.AM_E_INVAL
        self.st.set_remedy(on)
        return 0


@pytest.mark.parametrize("case", remedy_hold_cases.CASES, ids=lambda c: c.__name__)
def test_hand_derived_cases(am, orc, case):
    case(am, OracleDriver(am))


def _steps(rng, n, T, zmap, st_a, st_b, remedy_actions):
    """the same random calls on two oracle states, then a tick of each; yields both results"""
    for step in [0, 1, 1, 57, 1, 2, 60, 29, 1, 3600, 1, 31]:
        if step:
            fl = np.flatnonzero(st_a.since != timeout_oracle.hold_oracle.NOT_IN_FLIGHT)
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
    a = remedy_hold_oracle.State(zmap, cols, remedy=what != "remedy_hold_off")
    b = timeout_oracle.State(zmap, cols)
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
    for name in a.ocols:
        np.testing.assert_array_equal(a.ocols[name], b.ocols[name], err_msg=name)
    assert (a.rsince == remedy_hold_oracle.NONE).all() and seen > 1000
