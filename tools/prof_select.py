"""Sparse state queries (am_sweep_select) against the dense reads they replace, at BASELINE config 5's 10 M records with
the population of tools/run_sim.py (the hold in flight, the remedy hold, workflow timeouts on a tenth of the slots).
A simulated hour (am_sweep_simulate) puts runs of both kinds in flight; then a small submit budget and a few ticks
leave a backlog waiting for admission.  For each state, alternated in every round:

  select      s.select(state, cap=<the count>): one call, every match with its value
  count       the counting form (cap 0), before = INT64_MAX and before = T - 300
  dense       the dense query (in_flight, remedy_in_flight, deferred) followed by the numpy filter that gives the same list

Per form: device_ms, CUDA events on the handle's stream around the call (the passes and the copies to the host), and
host_ms, the whole call on the host clock (for `dense` with the filter).  The answers of select and dense are compared
once per state.  The card's name and power limit are read in the same run.  Prints one JSON object."""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tools", "amgen")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import run_sim  # noqa: E402

NONE = -(1 << 63)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--budget", type=int, default=2000)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    am = importlib.import_module("active-monitor_b200")
    import torch

    cols, sl, recs = run_sim.population(am, a.n, run_sim.SEED)
    T = run_sim.amgen.T0_DAY_START
    res = {"workload": f"config 5: {a.n} records after a simulated hour (hold in flight, remedy hold, a tenth with "
                       f"workflow timeouts), then ticks under a budget of {a.budget} per tick", "reps": a.reps}
    with am.Sweep(capacity=a.n) as s:
        s.load_range(0, cols)
        s.set_hold_in_flight(True)
        s.set_hold_remedy(True)
        s.upsert(sl, recs)
        s.simulate(T, 3600, am.SWEEP_BLOCKED, run_sim.SEED, run_sim.PARAMS)
        T += 3600
        s.set_submit_budget(a.budget)
        for step in (0, 1, 59, 1, 60):
            T += step
            s.tick(T)
        stream = torch.cuda.ExternalStream(s.stream)
        dense_of = {am.SEL_IN_FLIGHT: s.in_flight, am.SEL_REMEDY_IN_FLIGHT: s.remedy_in_flight,
                    am.SEL_WAITING: s.deferred}
        names = {am.SEL_IN_FLIGHT: "in_flight", am.SEL_REMEDY_IN_FLIGHT: "remedy_in_flight", am.SEL_WAITING: "waiting"}

        def timed(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            t0 = time.perf_counter()
            out = fn()
            host = (time.perf_counter() - t0) * 1e3
            e1.record(stream)
            torch.cuda.synchronize()
            return out, e0.elapsed_time(e1), host

        def dense_list(state):
            v = dense_of[state](0, a.n)
            hit = np.flatnonzero(v != NONE)
            return hit.astype(np.uint64), v[hit]

        res["states"] = {}
        for state, name in names.items():
            _, _, nm, old = s.select(state, cap=0)
            forms = {"select": lambda: s.select(state, cap=nm), "count": lambda: s.select(state, cap=0),
                     "count_older_than_300s": lambda: s.select(state, before=T - 300, cap=0),
                     "dense": lambda: dense_list(state)}
            got = s.select(state, cap=nm)
            want = dense_list(state)
            equal = bool(np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and got[2] == len(want[0])
                         and got[3] == (int(want[1].min()) if len(want[1]) else (1 << 63) - 1))
            t = {f: {"device_ms": [], "host_ms": []} for f in forms}
            for r in range(a.reps + 2):  # two rounds of warm-up
                for f, fn in forms.items():
                    _, dev, host = timed(fn)
                    if r >= 2:
                        t[f]["device_ms"].append(dev)
                        t[f]["host_ms"].append(host)
            res["states"][name] = {"n_match": nm, "oldest_age_s": T - old if nm else None, "equal": equal,
                                   **{f: {k: {"median": statistics.median(v), "min": min(v)} for k, v in d.items()}
                                      for f, d in t.items()}}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable: {e}"
    res.update({"card": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": q, "n_records": a.n})
    out = json.dumps(res, indent=1)
    print(out)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(out)


if __name__ == "__main__":
    main()
