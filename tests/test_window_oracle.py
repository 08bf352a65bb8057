"""The catch-up oracle (tests/window_oracle.py) rewrites records around a call of the C oracle's orc_sweep.  On a
window whose only minute start is T itself (or that holds none), its answer must be orc_sweep's at T: list,
statistics and every column, open and closed loop, on the adversarial population.  This pins the property the
composition relies on — nothing after the oracle's due decision depends on a record's kind or interval."""
import numpy as np
import pytest

import window_oracle
from adversarial import ZoneMap, population, zones_usable


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("T", [1789982100, 1789982100 + 37, 1790812800 + 13 * 86400 + 14 * 3600])
def test_window_oracle_is_orc_sweep_on_a_window_holding_only_T(am, orc, mode, T):
    zmap = ZoneMap()
    P = T - 59 if T % 60 == 0 else T - 20
    rng = np.random.default_rng(T % 997 + mode)
    cols = population(rng, 20_000, P, True, zmap.ids_of(zones_usable(P, T)))
    a = {k: v.copy() for k, v in cols.items()}
    b = {k: v.copy() for k, v in cols.items()}
    wi, wa, ws = window_oracle.sweep_window(zmap, a, P, T, mode=mode, seed=3)
    pi, pa, ps = zmap.sweep(b, T, mode=mode, seed=3)
    assert ws == ps
    np.testing.assert_array_equal(wi, pi)
    np.testing.assert_array_equal(wa, pa)
    for name in am.COLUMN_NAMES:
        np.testing.assert_array_equal(a[name], b[name], err_msg=name)
    assert ws["n_submit_hc"] > 1000 and ws["n_result_ok"] > 0
