"""Random call sequences through every entry point with workflow timeouts: tests/test_call_sequences_gpu.py's walks, with
a wf_timeout on most upserted records, against the same model (tests/handle_model.py, whose hold keeps the deadlines).
After every tick the walk also compares am_sweep_last_timed_out with the model's list."""
import zlib

import numpy as np
import pytest

from adversarial import ZoneMap, population
from test_call_sequences_gpu import WALKS, Walk, _capacity

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


class TimeoutWalk(Walk):
    def __init__(self, am, zmap, name, seed, capacity, base, T0):
        super().__init__(am, zmap, name, seed, capacity, base, T0)
        self.reached["timed_out"] = 0

    def records(self, k):
        recs = self.am.columns_to_records(population(self.rng, k, self.T, True, self.tz_ids))
        recs["wf_timeout"] = np.where(self.rng.random(k) < 0.3, 0, self.rng.integers(1, 240, k))
        return recs

    def tick(self, T, mode, every_column, entry=None):
        done = super().tick(T, mode, every_column, entry)
        got, want = self.s.last_timed_out(), self.m.last_timed_out()
        np.testing.assert_array_equal(got[0], want[0], err_msg=str(self.where))
        np.testing.assert_array_equal(got[1], want[1], err_msg=str(self.where))
        self.reached["timed_out"] += len(got[0])
        return done


@pytest.mark.parametrize("rep", [0, 1])
@pytest.mark.parametrize("k", range(len(WALKS)), ids=[w[3] for w in WALKS])
def test_random_call_sequences_with_timeouts_equal_the_model(am, zmap, k, rep):
    cap, base, T0, name = WALKS[k]
    cap = _capacity(k, cap)
    seed = zlib.crc32(f"timeout {name} {rep}".encode())
    T0 += 41 * rep
    walk = TimeoutWalk(am, zmap, name, seed, cap, base, T0)
    calls, reached = walk.run()
    print(f"\n{name}: capacity {cap}, base {base}, seed {seed}: {sum(calls.values())} calls, reached {reached}")
    assert reached["held"] > 0 and reached["nospace"] > 0, reached
