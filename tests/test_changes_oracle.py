"""The changed-set oracle (tests/changes_oracle.py) on the hand-derived cases, and the column diff it is built on."""
import numpy as np
import pytest

import changes_cases
import changes_oracle
from adversarial import ZoneMap
from handle_model import HandleModel


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


@pytest.mark.parametrize("case", changes_cases.CASES, ids=lambda c: c.__name__)
def test_hand_derived_cases(am, zmap, case):
    case(am, HandleModel(zmap, case.n, hold=case.hold is not None, remedy=case.hold == "remedy", track=True))


def test_masked_bits_and_anomaly():
    before = changes_oracle.empty_columns(4)
    before["flags"][:] = 2
    after = changes_oracle.snapshot(before)
    after["flags"][0] |= (1 << 4) | (1 << 12)  # a pending bit and a carry bit: not a change
    after["flags"][1] |= 1 << 10                # the timer: a change
    after["failed"][2] += 1                     # reported ANOMALY: not listed
    after["failed"][3] += 1                     # ANOMALY and STOPPED: listed
    got = changes_oracle.changed(before, after, np.array([102, 103]), np.array([0x80, 0x84]), shard_base=100)
    assert got.tolist() == [101, 103]
