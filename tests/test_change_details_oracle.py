"""The change-details oracle (tests/change_details_oracle.py) on the hand-derived cases."""
import numpy as np
import pytest

import change_details_cases
import change_details_oracle
from adversarial import ZoneMap
from handle_model import HandleModel


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


@pytest.mark.parametrize("case", change_details_cases.CASES, ids=lambda c: c.__name__)
def test_hand_derived_cases(am, zmap, case):
    case(am, HandleModel(zmap, case.n, hold=case.hold is not None, remedy=case.hold == "remedy", track=True, details=True))


def test_applied_of_maps_every_posted_bit():
    f = np.array([0, 1 << 4, 1 << 5, 1 << 6, (1 << 6) | (1 << 7), (1 << 5) | (1 << 6) | (1 << 7)], np.uint32)
    assert change_details_oracle.applied_of(f).tolist() == [0, 0x01, 0x02, 0x10, 0x08, 0x0A]
