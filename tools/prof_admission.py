"""Submit budget (am_sweep_set_submit_budget) on the config-2 population (10 M records by default), hold in flight and
workflow timeouts on: a handle that never sets a budget against one at budgets of 1 M, 100 k and 10 k per tick,
alternated in every round.  Device-resident ticks (am_sweep_tick_device, as in bench.py's timed loop), three cases:
  clean      an on-minute tick from a clean state (the hold toggled: nothing in flight, nothing waiting);
  idle       the tick one second after an unlimited on-minute tick: every due record is held, nothing waits;
  overload   the tick one second after a budgeted on-minute tick: millions of checks wait and the interval ones are due
             again (for the unlimited handle: the same tick as idle).
Step time: CUDA events around the call.  The admission passes' own time: the adm_* kernels in a torch.profiler capture of
one more round (a pass of its own).  Prints one JSON object, with the card's name and power limit read in the same run."""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools", "amgen")):
    sys.path.insert(0, p)
import amgen  # noqa: E402
import numpy as np  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=10_000_000)
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--out", default="")
a = ap.parse_args()
am = importlib.import_module("active-monitor_b200")
import torch  # noqa: E402

T0 = amgen.T0_MON_0915  # on the minute
cols = amgen.fill(2, 2, 0, a.n, T0, am.load().am_healthcheck_classify)
dev = torch.device("cuda", 0)
d_idx = torch.empty(a.n, dtype=torch.int32, device=dev)
d_act = torch.empty(a.n, dtype=torch.uint8, device=dev)
d_cnt = torch.zeros(1, dtype=torch.int32, device=dev)
d_st = torch.zeros(16, dtype=torch.int64, device=dev)
stream = torch.cuda.current_stream()
BUDGETS = [None, 1_000_000, 100_000, 10_000]
CASES = ("clean", "idle", "overload")


def name(b):
    return "unlimited" if b is None else str(b)


step = {(name(b), c): [] for b in BUDGETS for c in CASES}
adm_us = {(name(b), c): 0.0 for b in BUDGETS for c in CASES}
emitted, backlog = {}, {}
handles = {}
try:
    for b in BUDGETS[:2]:  # one handle without the admission state, one that gets every finite budget
        s = am.Sweep(capacity=a.n)
        s.load_range(0, cols)
        s.set_hold_in_flight(True)
        rec = am.columns_to_records({k: v[:1] for k, v in cols.items()})
        rec["wf_timeout"] = 300
        s.upsert([0], rec)  # (the timeout state: every submission gets a deadline)
        handles[b is None] = s

    def tick(s, T):
        s.tick_device(T, 0, d_idx.data_ptr(), d_act.data_ptr(), a.n, d_cnt.data_ptr(), d_st.data_ptr(), stream.cuda_stream)

    def run_round(r, record):
        T = T0 + 7 * 86400 * (r + 1)
        for b in BUDGETS:
            s = handles[b is None]
            for c in CASES:
                s.set_hold_in_flight(False)
                s.set_hold_in_flight(True)  # nothing in flight, nothing waiting, the budget unlimited
                if c != "clean":  # the on-minute tick before: unlimited for idle, budgeted for overload
                    if c == "overload":
                        s.set_submit_budget(b)
                    tick(s, T)
                s.set_submit_budget(b)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                tick(s, T if c == "clean" else T + 1)
                e1.record(stream)
                torch.cuda.synchronize()
                if record:
                    step[(name(b), c)].append(e0.elapsed_time(e1))
                    emitted[(name(b), c)] = int(d_st[1].item())
                    backlog[(name(b), c)] = s.last_admission()["n_deferred"] if b is not None else 0

    for r in range(a.reps + 2):  # the first two rounds warm up
        run_round(r, r >= 2)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run_round(a.reps + 2, False)
    # kernels of the capture in issue order: attribute each adm_* kernel to the case whose timed tick launched it
    # (one profiled round: the budgeted handle's cases in BUDGETS x CASES order, two ticks for idle / overload)
    kern = [(e.name, e.device_time) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    adm = [us for nm, us in kern if "adm_" in nm and "next_due" not in nm and "gather" not in nm]
    per_tick = 6
    ticks = [(name(b), c) for b in BUDGETS[1:] for c in CASES for _ in range(1 if c == "clean" else 2)]
    for k, key in enumerate(ticks):
        chunk = adm[k * per_tick:(k + 1) * per_tick]
        if len(chunk) == per_tick:
            adm_us[key] = sum(chunk)  # (idle, overload: the second of their two ticks, the timed one, wins)
finally:
    for s in handles.values():
        s.close()

try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:  # noqa: BLE001
    q = f"nvidia-smi unavailable: {e}"
res = {"card": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": q, "n_records": a.n, "reps": a.reps,
       "ticks": {}}
for (b, c), v in step.items():
    res["ticks"][f"{b}/{c}"] = {"step_ms_median": statistics.median(v), "step_ms_min": min(v),
                                "n_emitted": emitted[(b, c)], "waiting_after": backlog[(b, c)],
                                "admission_passes_us": round(adm_us[(b, c)], 1)}
out = json.dumps(res, indent=1)
print(out)
if a.out:
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        f.write(out)
