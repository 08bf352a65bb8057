"""The hold-in-flight oracle (tests/hold_oracle.py) rewrites held records around a call of the C oracle's orc_sweep (or
of the window oracle).  With nothing held its answer is orc_sweep's: list, statistics and every column.  With holds, a
held record differs from the plain tick only by losing SUBMIT_HC: every other entry, action and column is the plain
tick's, and the statistics differ by exactly the lost submissions."""
import numpy as np
import pytest

import hold_oracle
import window_oracle
from adversarial import ZoneMap, population, zones_usable

TS = [1789982100, 1789982100 + 37, 1790812800 + 13 * 86400 + 14 * 3600]


@pytest.mark.parametrize("catch_up", [False, True])
@pytest.mark.parametrize("T", TS)
def test_nothing_held_is_the_plain_tick(am, orc, T, catch_up):
    zmap = ZoneMap()
    P = T - 700
    rng = np.random.default_rng(T % 991)
    cols = population(rng, 20_000, P, True, zmap.ids_of(zones_usable(P, T)))
    a = {k: v.copy() for k, v in cols.items()}
    b = {k: v.copy() for k, v in cols.items()}
    since = hold_oracle.none_in_flight(20_000)
    got = hold_oracle.sweep(zmap, a, since, T, P=P if catch_up else None, seed=3)
    want = window_oracle.sweep_window(zmap, b, P, T, seed=3) if catch_up else zmap.sweep(b, T, seed=3)
    assert got[2] == want[2]
    np.testing.assert_array_equal(got[0], want[0])
    np.testing.assert_array_equal(got[1], want[1])
    for name in am.COLUMN_NAMES:
        np.testing.assert_array_equal(a[name], b[name], err_msg=name)
    sub = (want[1] & am.ACT_SUBMIT_HC) != 0
    np.testing.assert_array_equal(np.flatnonzero(since == T), np.sort(want[0][sub].astype(np.int64)))
    assert want[2]["n_submit_hc"] > 1000


@pytest.mark.parametrize("catch_up", [False, True])
@pytest.mark.parametrize("T", TS)
def test_a_held_record_only_loses_its_submission(am, orc, T, catch_up):
    zmap = ZoneMap()
    P = T - 700
    n = 20_000
    rng = np.random.default_rng(T % 983 + 1)
    cols = population(rng, n, P, True, zmap.ids_of(zones_usable(P, T)))
    # a third of the slots submitted at some earlier second, some of them since released by a later finishedAt
    since = hold_oracle.none_in_flight(n)
    pick = rng.random(n) < 0.33
    since[pick] = cols["finished_at"][pick] + rng.integers(-2, 3, n)[pick]
    a = {k: v.copy() for k, v in cols.items()}
    b = {k: v.copy() for k, v in cols.items()}
    h = hold_oracle.held(a, since)
    since0 = since.copy()
    gi, ga, gs = hold_oracle.sweep(zmap, a, since, T, P=P if catch_up else None, seed=5)
    wi, wa, ws = window_oracle.sweep_window(zmap, b, P, T, seed=5) if catch_up else zmap.sweep(b, T, seed=5)
    for name in am.COLUMN_NAMES:
        np.testing.assert_array_equal(a[name], b[name], err_msg=name)
    plain = dict(zip(wi.tolist(), wa.tolist()))
    got = dict(zip(gi.tolist(), ga.tolist()))
    lost = 0
    for i, act in plain.items():
        if h[i] and act & am.ACT_SUBMIT_HC:
            lost += 1
            rest = act & ~am.ACT_SUBMIT_HC
            assert got.get(i, 0) == rest, i
        else:
            assert got.get(i) == act, i
    assert set(got) <= set(plain)
    assert lost > 100
    assert gs["n_submit_hc"] == ws["n_submit_hc"] - lost and gs["n_emitted"] <= ws["n_emitted"]
    # held STOPPED / PARSE_ERROR records keep their actions
    kinds = b["flags"] & np.uint32(am.KIND_MASK)
    assert any(h[i] and kinds[i] in (am.KIND_STOPPED, am.KIND_PARSE_ERROR) for i in got)
    # since: T for every submission, unchanged elsewhere
    sub = np.zeros(n, dtype=bool)
    sub[[i for i, v in got.items() if v & am.ACT_SUBMIT_HC]] = True
    np.testing.assert_array_equal(since[sub], T)
    np.testing.assert_array_equal(since[~sub], since0[~sub])
