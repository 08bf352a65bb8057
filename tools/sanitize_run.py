"""Small driver for compute-sanitizer: every kernel variant (open/closed loop, on/off
minute), staged upsert/remove/post_result, read-by-index, on-device Next(), and one sparse state query per state."""
import importlib, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools", "amgen")):
    sys.path.insert(0, p)
import numpy as np
import amgen
am = importlib.import_module("active-monitor_b200")
n, T0 = 70_001, amgen.T0_MON_0915
cols = amgen.fill(3, 3, 0, n, T0, am.load().am_healthcheck_classify)
with am.Sweep(capacity=n + 500) as s:
    s.load_range(0, cols)
    s.set_seed(3)
    recs = am.columns_to_records(cols)
    tot = 0
    for k, (T, mode) in enumerate([(T0, 0), (T0 + 1, 0), (T0 + 60, 1), (T0 + 61, 1), (T0 + 62, 3)]):
        s.upsert(np.arange(n, n + 50) + k, recs[:50])
        s.remove([5 + k, 9000 + k])
        s.post_result(np.arange(100, 4000, 7), np.full(558, 1 + k % 2, np.uint8), np.full(558, k % 3, np.uint8))
        idx, act, st = s.tick(T, mode=mode)
        tot += st["n_emitted"]
    s.read(np.arange(0, n, 97))
    s.repeat_after_sec(T0, 0, 5000)
    s.run_ticks(T0 + 100, 5, mode=1, seed=3)
    s.set_hold_in_flight(True)
    s.set_hold_remedy(True)
    s.set_submit_budget(100)
    s.tick(T0 + 200)
    for state in (am.SEL_IN_FLIGHT, am.SEL_REMEDY_IN_FLIGHT, am.SEL_WAITING):
        s.select(state, 3, n - 10, T0 + 200, cap=1000)
print("sanitize_run ok", tot)
