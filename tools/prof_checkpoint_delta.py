"""Delta checkpoints at BASELINE config 5's 10 M records, with the population and switches of tools/prof_checkpoint.py
(the hold in flight, the remedy hold, workflow timeouts on a tenth of the slots, status changes with details), after a
simulated hour.  A chain's root is taken and restored into a standby; then, for simulated periods of 1, 10 and 60 s
between links, the source simulates one period and takes a delta that the standby applies.  Measured per period,
each repeated:

  n_changed, delta_bytes  the slots a delta carries and its length, against the full blob's (full_bytes)
  delta_ms                the whole am_sweep_checkpoint_delta call (drain, diff, compaction, pack, copy, commit)
  diff_ms                 delta_diff_kernel's device time (torch.profiler, one call per period)
  guard_ms                the tick guard held by the call: a second thread ticks the source in a loop during it; the
                          span from its first to its last AM_E_BUSY answer (as in tools/prof_checkpoint.py)
  restore_delta_ms        the whole am_sweep_restore_delta call on the standby

The card's name and power limit are read in the same run.  Prints one JSON object."""
import argparse
import importlib
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tools", "amgen")):
    sys.path.insert(0, p)
import run_sim  # noqa: E402
from prof_checkpoint import busy_span, handle, retry_busy  # noqa: E402


def standby(am, n):
    t = am.Sweep(capacity=n)
    t.set_hold_in_flight(True)
    t.set_hold_remedy(True)
    t.set_track_changes(True)
    t.set_change_details(True)
    return t


def diff_ms(am, s):
    """one delta under torch.profiler: (the delta, delta_diff_kernel's device ms)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = s.checkpoint_delta()
    ms = sum(e.device_time_total for e in prof.key_averages() if "delta_diff_kernel" in e.key) / 1e3
    return out, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--periods", default="1,10,60")
    a = ap.parse_args()
    am = importlib.import_module("active-monitor_b200")
    import torch  # noqa: F401  (CUDA context for the profiler)
    cols, sl, recs = run_sim.population(am, a.n, run_sim.SEED)
    s = handle(am, cols, sl, recs)
    T = run_sim.amgen.T0_DAY_START
    s.simulate(T, 3600, am.SWEEP_BLOCKED, run_sim.SEED, run_sim.PARAMS)
    T += 3600
    t0 = time.perf_counter()
    root = s.checkpoint_chain(0, a.n)
    chain_ms = (time.perf_counter() - t0) * 1e3
    sb = standby(am, a.n)
    sb.restore(root)
    out = {"workload": f"config 5: {a.n} records after a simulated hour (hold in flight, remedy hold, a tenth with "
                       f"workflow timeouts, status changes with details); a chain over every slot, a delta after each "
                       f"simulated period, applied to a standby",
           "card": run_sim.card(), "full_bytes": len(root), "checkpoint_chain_ms": round(chain_ms, 2), "periods": {}}
    for period in (int(x) for x in a.periods.split(",")):
        rows = {k: [] for k in ("n_changed", "delta_bytes", "delta_ms", "restore_delta_ms")}
        for _ in range(a.repeat):
            s.simulate(T, period, am.SWEEP_BLOCKED, run_sim.SEED, run_sim.PARAMS)
            T += period
            t0 = time.perf_counter()
            d, k = s.checkpoint_delta()
            rows["delta_ms"].append((time.perf_counter() - t0) * 1e3)
            rows["n_changed"].append(k)
            rows["delta_bytes"].append(len(d))
            t0 = time.perf_counter()
            sb.restore_delta(d)
            rows["restore_delta_ms"].append((time.perf_counter() - t0) * 1e3)
        # the device time of the diff, and the guard a concurrent ticker meets (both links go to the standby as well)
        s.simulate(T, period, am.SWEEP_BLOCKED, run_sim.SEED, run_sim.PARAMS)
        T += period
        (d, _), dms = diff_ms(am, s)
        sb.restore_delta(d)
        (d, _), guard = busy_span(am, s, T, lambda: retry_busy(am, lambda: s.checkpoint_delta()))
        sb.restore_delta(d)
        T += 1
        out["periods"][str(period)] = {
            "n_changed_median": int(statistics.median(rows["n_changed"])),
            "delta_bytes_median": int(statistics.median(rows["delta_bytes"])),
            "delta_over_full": round(statistics.median(rows["delta_bytes"]) / len(root), 5),
            "delta_ms_median": round(statistics.median(rows["delta_ms"]), 2),
            "restore_delta_ms_median": round(statistics.median(rows["restore_delta_ms"]), 2),
            "diff_ms": round(dms, 3), "guard_ms": round(guard, 2), "raw": rows}
    sb.restore_delta(s.checkpoint_delta()[0])  # (the ticks of the last guard measurement)
    out["standby_matches_source"] = sb.checkpoint(0, a.n) == s.checkpoint(0, a.n)
    print(json.dumps(out))
    s.close()
    sb.close()


if __name__ == "__main__":
    main()
