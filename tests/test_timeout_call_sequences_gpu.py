"""Random call sequences through every entry point with workflow timeouts: tests/test_call_sequences_gpu.py's walks, with
a wf_timeout on most upserted records, against SequenceModel extended by the timeout oracle (tests/timeout_oracle.py).
After every tick the walk also compares am_sweep_last_timed_out with the model's list."""
import zlib

import numpy as np
import pytest

import timeout_oracle
from adversarial import ZoneMap, population
from sequence_model import CLOSED_LOOP, E_INVAL, E_RANGE, Refused, SequenceModel
from test_call_sequences_gpu import WALKS, Walk, _capacity

pytestmark = pytest.mark.gpu

EMPTY = (np.zeros(0, dtype=np.uint64), np.zeros(0, dtype=np.int64))


@pytest.fixture(scope="module")
def zmap(am, orc):
    return ZoneMap()


class TimeoutModel(SequenceModel):
    """SequenceModel plus W and D per slot and the last tick's timed-out list"""

    def __init__(self, zmap, capacity, shard_base=0, seed=0):
        super().__init__(zmap, capacity, shard_base, seed)
        self.wf = np.zeros(capacity, dtype=np.int32)
        self.deadline = timeout_oracle.no_deadlines(capacity)
        self.last_timed = EMPTY

    def upsert(self, idx, recs):
        super().upsert(idx, recs)
        idx = np.asarray(idx, dtype=np.int64)
        _, rev = np.unique(idx[::-1], return_index=True)
        last = len(idx) - 1 - rev
        self.wf[idx[last]] = recs["wf_timeout"][last]

    def remove(self, idx):
        super().remove(idx)
        self.deadline[np.asarray(idx, dtype=np.int64)] = timeout_oracle.NO_DEADLINE

    def load(self, first, cols):
        super().load(first, cols)
        n = len(cols["flags"])
        self.wf[first:first + n] = 0
        self.deadline[first:first + n] = timeout_oracle.NO_DEADLINE

    def set_hold(self, on):
        if on and not self.hold:
            self.deadline[:] = timeout_oracle.NO_DEADLINE
        super().set_hold(on)

    def _timed_sweep(self, cols, since, deadline, T, P, mode, seed):
        timed = timeout_oracle.expire(cols, since, deadline, T, self.shard_base)
        out = self._sweep(cols, since, T, P, mode, seed)
        loc = np.asarray(out[0], dtype=np.int64)[(np.asarray(out[1]) & timeout_oracle.ACT_SUBMIT_HC) != 0] - self.shard_base
        w = self.wf[loc].astype(np.int64)
        deadline[loc] = np.where(w > 0, T + w, timeout_oracle.NO_DEADLINE)
        return out, timed

    def tick(self, T, mode):
        if self.hold and (mode & CLOSED_LOOP):
            raise Refused(E_INVAL)
        P = self.window_of(T, mode)
        if P is not None and T - P > 86400:
            raise Refused(E_RANGE)
        if not self.hold:
            self.last_timed = EMPTY
            return super().tick(T, mode)
        h = self.hwm
        out, self.last_timed = self._timed_sweep(self.view(), self.since[:h], self.deadline[:h], T, P, mode, self.seed)
        self.P = T
        return out

    def run_ticks(self, T0, n, mode, seed):
        rows = super().run_ticks(T0, n, mode, seed)
        self.last_timed = EMPTY
        return rows

    def first_active_tick(self, T, horizon):
        if not self.hold:
            return super().first_active_tick(T, horizon)
        h = self.hwm
        cols = {k: v.copy() for k, v in self.view().items()}
        since, deadline = self.since[:h].copy(), self.deadline[:h].copy()
        for t in range(T + 1, T + horizon + 1):
            (_, _, st), timed = self._timed_sweep(cols, since, deadline, t, None, 0, 0)
            if st["n_emitted"] or len(timed[0]) or any(st[k] for k in ("n_result_ok", "n_result_fail", "n_remedy_ok",
                                                                        "n_remedy_fail")):
                return t
        return None


class TimeoutWalk(Walk):
    def __init__(self, am, zmap, name, seed, capacity, base, T0):
        super().__init__(am, zmap, name, seed, capacity, base, T0)
        self.m = TimeoutModel(zmap, capacity, base, seed=seed)
        self.reached["timed_out"] = 0

    def records(self, k):
        recs = self.am.columns_to_records(population(self.rng, k, self.T, True, self.tz_ids))
        recs["wf_timeout"] = np.where(self.rng.random(k) < 0.3, 0, self.rng.integers(1, 240, k))
        return recs

    def tick(self, T, mode, every_column, entry=None):
        done = super().tick(T, mode, every_column, entry)
        got, want = self.s.last_timed_out(), self.m.last_timed
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
