"""Spec updates (am_sweep_update_spec) on the config-2 population (10 M records by default), device-resident ticks
(am_sweep_tick_device, as in bench.py's timed loop), alternated in every round:
  drain        a tick whose drain holds one call per record: upserts of the records as they were loaded, spec updates
               with the same specs (every record's status kept, no plane rebuilt), spec updates with another seed's
               specs (kinds, masks and zones change: planes rebuilt);
  echo         a tick whose drain holds 1.5 M spec updates of random records with unchanged specs (the status echoes of
               one config-2 tick's write-back) against the same tick with an empty drain;
  staging      the host time of one am_sweep_upsert / am_sweep_update_spec call of 1 M records.
Every round reloads the records first (not timed).  Tick time: the host clock around the call and a device
synchronise (the drain's copies and the kernels), median over the rounds.  The drain kernels' own times: a
torch.profiler capture of one more round (a pass of its own).  Prints one JSON object, with the card's name and power
limit read in the same run."""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools", "amgen")):
    sys.path.insert(0, p)
import amgen  # noqa: E402
import numpy as np  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=10_000_000)
ap.add_argument("--echo", type=int, default=1_500_000)
ap.add_argument("--stage", type=int, default=1_000_000)
ap.add_argument("--reps", type=int, default=7)
ap.add_argument("--out", default="")
a = ap.parse_args()
am = importlib.import_module("active-monitor_b200")
import torch  # noqa: E402

T0 = amgen.T0_MON_0915 + 17  # off the minute: the tick reads no masks, so the drain is most of it
classify = am.load().am_healthcheck_classify
cols = amgen.fill(2, 2, 0, a.n, T0, classify)
same = am.columns_to_records(cols)
other = am.columns_to_records(amgen.fill(2, 3, 0, a.n, T0, classify))
slots = np.arange(a.n, dtype=np.uint64)
rng = np.random.default_rng(1)
echo_idx = rng.choice(a.n, a.echo, replace=False).astype(np.uint64)
echo_recs = same[echo_idx.astype(np.int64)]
dev = torch.device("cuda", 0)
d_idx = torch.empty(a.n, dtype=torch.int32, device=dev)
d_act = torch.empty(a.n, dtype=torch.uint8, device=dev)
d_cnt = torch.zeros(1, dtype=torch.int32, device=dev)
d_st = torch.zeros(16, dtype=torch.int64, device=dev)
stream = torch.cuda.current_stream()

DRAIN = {"upsert": lambda s: s.upsert(slots, same), "spec_same": lambda s: s.update_spec(slots, same),
         "spec_other": lambda s: s.update_spec(slots, other)}
ECHO = {"echo_1.5M": lambda s: s.update_spec(echo_idx, echo_recs), "empty": lambda s: None}
times = {k: [] for k in list(DRAIN) + list(ECHO)}
stage_ms = {"upsert": [], "update_spec": []}
DRAIN_KERNELS = ("mark_ops", "apply_state_ops", "apply_spec_ops", "build_planes_dirty", "clear_marks")
kern_us = {}


def timed_tick(s, T):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    s.tick_device(T, 0, d_idx.data_ptr(), d_act.data_ptr(), a.n, d_cnt.data_ptr(), d_st.data_ptr(), stream.cuda_stream)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def run_round(s, r, record):
    T = T0 + 7 * 86400 * (r + 1)
    for name, call in list(DRAIN.items()) + list(ECHO.items()):
        s.load_range(0, cols)
        timed_tick(s, T - 60)  # (a tick before: the drain of the load is not in the timed one)
        call(s)
        ms = timed_tick(s, T)
        if record:
            times[name].append(ms)
    for name, call in (("upsert", lambda: s.upsert(slots[:a.stage], same[:a.stage])),
                       ("update_spec", lambda: s.update_spec(slots[:a.stage], same[:a.stage]))):
        t0 = time.perf_counter()
        call()
        ms = (time.perf_counter() - t0) * 1e3
        timed_tick(s, T + 1)
        if record:
            stage_ms[name].append(ms)


s = am.Sweep(capacity=a.n)
try:
    for r in range(a.reps + 1):  # the first round warms up
        run_round(s, r, r >= 1)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run_round(s, a.reps + 1, False)
    # the drain kernels of the capture in issue order, attributed to the timed tick of each case (the second of its
    # two ticks; a load's drain launches none of them): one group per case with a drain
    kern = [(e.name, e.device_time) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    groups, cur = [], None
    for nm, us in kern:
        k = next((d for d in DRAIN_KERNELS if d in nm), None)
        if k is None:
            if cur is not None:
                groups.append(cur)
                cur = None
            continue
        cur = cur or {}
        cur[k] = cur.get(k, 0.0) + us
    if cur is not None:
        groups.append(cur)
    with_drain = list(DRAIN) + ["echo_1.5M"]
    # per case in order: its timed tick's drain; then the two staging calls' drains (not reported)
    for name, g in zip(with_drain, groups):
        kern_us[name] = {k: round(v, 1) for k, v in g.items()}
finally:
    s.close()

try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:  # noqa: BLE001
    q = f"nvidia-smi unavailable: {e}"
res = {"card": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": q, "n_records": a.n, "echo": a.echo,
       "reps": a.reps, "tick_ms": {}, "staging_ms_per_1M": {}, "drain_kernels_us": kern_us}
for k, v in times.items():
    res["tick_ms"][k] = {"median": round(statistics.median(v), 3), "min": round(min(v), 3)}
for k, v in stage_ms.items():
    res["staging_ms_per_1M"][k] = round(statistics.median(v) * 1e6 / a.stage, 3)
out = json.dumps(res, indent=1)
print(out)
if a.out:
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        f.write(out)
