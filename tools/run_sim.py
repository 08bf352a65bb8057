"""A simulated day of the recommended controller configuration (INTEGRATION.md §3: the hold in flight, the remedy hold
and workflow timeouts on) at BASELINE config 5's 10 M records, through am_sweep_simulate.

Population: config 5's records (tools/amgen), a seeded fraction of the slots upserted again with a non-zero
wf_timeout; both holds are turned on before the first tick.  The run is blocked (sweep_block.cuh); with
--compare-unblocked the same day runs tick by tick on a second handle and every statistics row, every simulated row,
all sixteen columns and both in-flight answers are compared bit for bit.  --repeat alternates the two paths on fresh
handles and reports the per-tick device time of each run.  The card's name and power limit are read in the same run.
Prints one JSON object."""
import argparse
import importlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools", "amgen")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import amgen  # noqa: E402

SEED = 5
PARAMS = (30, 600, 60, 900)  # health-check and remedy workflow durations, seconds (min, max)


def population(am, n, seed, timeout_fraction=0.1):
    """config 5's columns, and the slots re-upserted with a workflow timeout (records of their own)"""
    cols = amgen.fill(5, seed, 0, n, amgen.T0_DAY_START, am.load().am_healthcheck_classify)
    rng = np.random.default_rng(seed)
    sl = np.sort(rng.choice(n, int(n * timeout_fraction), replace=False))
    recs = am.columns_to_records({k: v[sl] for k, v in cols.items()})
    recs["wf_timeout"] = rng.integers(60, 900, len(sl))
    return cols, sl, recs


def run(am, cols, sl, recs, seconds, blocked, seed=SEED, params=PARAMS):
    """(stats rows, sim rows, device ms, columns, in flight, remedy in flight) of one simulated run on a fresh handle"""
    n = len(cols["flags"])
    with am.Sweep(capacity=n) as s:
        s.load_range(0, cols)
        s.set_hold_in_flight(True)
        s.set_hold_remedy(True)
        s.upsert(sl, recs)
        rows, sim = s.simulate(amgen.T0_DAY_START, seconds, am.SWEEP_BLOCKED if blocked else 0, seed, params)
        ms = s.last_kernel_ms
        return rows, sim, ms, s.read_range(0, n), s.in_flight(0, n), s.remedy_in_flight(0, n)


def compare(am, n=10_000_000, seconds=86_400, seed=SEED):
    cols, sl, recs = population(am, n, seed)
    a = run(am, cols, sl, recs, seconds, True, seed)
    b = run(am, cols, sl, recs, seconds, False, seed)
    fields = am.abi.STAT_FIELDS
    equal = {"stats": all(np.array_equal(a[0][f], b[0][f]) for f in fields), "sim": bool(np.array_equal(a[1], b[1])),
             "columns": all(np.array_equal(a[3][c], b[3][c]) for c in am.COLUMN_NAMES),
             "in_flight": bool(np.array_equal(a[4], b[4])), "remedy_in_flight": bool(np.array_equal(a[5], b[5]))}
    sim = a[1]
    return {"equal": all(equal.values()), "which": equal, "blocked_us_per_tick": a[2] * 1e3 / seconds,
            "unblocked_us_per_tick": b[2] * 1e3 / seconds, "peak_in_flight": int(sim["n_in_flight"].max()),
            "peak_remedy_in_flight": int(sim["n_remedy_in_flight"].max()), "timed_out": int(sim["n_timed_out"].sum()),
            "remedy_timed_out": int(sim["n_remedy_timed_out"].sum()), "remedies": int(a[0]["n_run_remedy"].sum()),
            "submits": int(a[0]["n_submit_hc"].sum())}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or q.stderr.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--seconds", type=int, default=86_400)
    ap.add_argument("--compare-unblocked", action="store_true")
    ap.add_argument("--repeat", type=int, default=0, help="alternate blocked and unblocked runs this many times each")
    a = ap.parse_args()
    am = importlib.import_module("active-monitor_b200")
    out = {"workload": f"config 5: {a.n} records, {a.seconds} simulated one-second ticks from 2026-09-21T00:00:00Z, "
                       f"hold in flight + remedy hold, a tenth of the slots with workflow timeouts of 60-899 s, "
                       f"durations {PARAMS} s, seed {SEED}",
           "card": card()}
    if a.compare_unblocked:
        out["compare"] = compare(am, a.n, a.seconds)
    if a.repeat:
        cols, sl, recs = population(am, a.n, SEED)
        times = {"blocked": [], "unblocked": []}
        for _ in range(a.repeat):
            for blocked in (True, False):
                ms = run(am, cols, sl, recs, a.seconds, blocked)[2]
                times["blocked" if blocked else "unblocked"].append(ms * 1e3 / a.seconds)
        out["us_per_tick"] = times
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
