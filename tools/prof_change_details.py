"""The cost of change details (am_sweep_set_change_details): two handles loaded alike with status changes tracked,
`track` (details off) and `details` (details on), alternated in every round; 10 M records by default.

Part 1, device-resident ticks (am_sweep_tick_device, as in bench.py's timed loop), medians over the rounds:
  sparse  config 2: Succeeded posted on ~2 % of the records before the timed tick (the drain's result kernel applies it);
  dense   config 3: its 75 % pending results (50 % Failed, 25 % Succeeded, remedy outcomes) posted before the timed tick
          (more than an eighth of the records: applied inside the sweep).
Kernel time: sweep_tick_kernel between CUDA events (am_sweep_set_profiling, a pass of its own).  Step time: CUDA events
around the whole call, in the other pass.
Part 2, the host time of am_sweep_last_change_details after each `details` tick of part 1, beside that of
am_sweep_last_changes for the eight status columns.

Prints one JSON object, with the card's name and power limit read in the same run."""
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
ap.add_argument("--reps", type=int, default=30)
ap.add_argument("--out", default="")
a = ap.parse_args()
am = importlib.import_module("active-monitor_b200")
import torch  # noqa: E402

STATUS = ["flags", "finished_at", "success", "failed", "remedy_success", "remedy_failed", "remedy_total",
          "remedy_finished_at"]
T0 = amgen.T0_MON_0915  # on the minute
HANDLES = ("track", "details")
dev = torch.device("cuda", 0)
d_idx = torch.empty(a.n, dtype=torch.int32, device=dev)
d_act = torch.empty(a.n, dtype=torch.uint8, device=dev)
d_cnt = torch.zeros(1, dtype=torch.int32, device=dev)
d_st = torch.zeros(16, dtype=torch.int64, device=dev)
stream = torch.cuda.current_stream()
rng = np.random.default_rng(7)
res = {"n_records": a.n, "reps": a.reps, "device_ticks": {}, "read_host_ms": {}}


def tick(s, T):
    s.tick_device(T, 0, d_idx.data_ptr(), d_act.data_ptr(), a.n, d_cnt.data_ptr(), d_st.data_ptr(), stream.cuda_stream)


def posts_of(config, cols):
    """config 2: Succeeded on ~2 % of the records; config 3: every pending result of the population"""
    if config == 2:
        sl = np.flatnonzero(rng.random(a.n) < 0.02).astype(np.uint64)
        return sl, np.full(len(sl), am.PHASE_SUCCEEDED, np.uint8), None
    fl = cols["flags"]
    sl = np.flatnonzero(fl & (am.F_PENDING_OK | am.F_PENDING_FAIL | am.F_REMEDY_PENDING)).astype(np.uint64)
    f = fl[sl]
    ph = np.where(f & am.F_PENDING_OK, 1, np.where(f & am.F_PENDING_FAIL, 2, 0)).astype(np.uint8)
    rp = np.where(f & am.F_REMEDY_PENDING, np.where(f & am.F_REMEDY_OUTCOME_OK, 1, 2), 0).astype(np.uint8)
    return sl, ph, rp


def timed_host(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


for config, part in ((2, "sparse"), (3, "dense")):
    cols = amgen.fill(config, config, 0, a.n, T0, am.load().am_healthcheck_classify)
    posts = posts_of(config, cols)
    clear = ~np.uint32(am.F_PENDING_OK | am.F_PENDING_FAIL | am.F_REMEDY_PENDING | am.F_REMEDY_OUTCOME_OK)
    cols["flags"] &= clear
    kern = {k: [] for k in HANDLES}
    step = {k: [] for k in HANDLES}
    host_det, host_status, listed = [], [], []
    with am.Sweep(capacity=a.n) as track, am.Sweep(capacity=a.n) as details:
        sw = {"track": track, "details": details}
        for s in (track, details):
            s.set_track_changes(True)
        details.set_change_details(True)
        for s in (track, details):
            s.load_range(0, cols)
        for profiled in (True, False):
            for r in range(a.reps + 2):  # the first two rounds warm up
                T = T0 + 86400 * (r + 1) + (0 if profiled else 3600)
                for k in HANDLES:
                    s = sw[k]
                    if config == 3:  # the step consumes its results: the same population every round
                        s.load_range(0, cols)
                    s.post_result(*posts)
                    s.set_profiling(profiled)
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    tick(s, T)
                    e1.record(stream)
                    torch.cuda.synchronize()
                    sweep_ms = s.last_profile()[0] if profiled else None
                    s.set_profiling(False)
                    if r < 2:
                        continue
                    if profiled:
                        kern[k].append(sweep_ms)
                    else:
                        step[k].append(e0.elapsed_time(e1))
                        if k == "details":
                            ms, (idx, _) = timed_host(lambda: s.last_change_details())
                            host_det.append(ms)
                            listed.append(len(idx))
                            ms, _ = timed_host(lambda: s.last_changes(names=STATUS))
                            host_status.append(ms)
    for k in HANDLES:
        res["device_ticks"][f"{part}/{k}"] = {"config": config, "posted": int(len(posts[0])),
                                              "sweep_kernel_ms_median": statistics.median(kern[k]),
                                              "step_ms_median": statistics.median(step[k]),
                                              "step_ms_min": min(step[k]), "step_ms_max": max(step[k])}
    res["read_host_ms"][part] = {"listed": int(statistics.median(listed)),
                                 "last_change_details_median": statistics.median(host_det),
                                 "last_changes_status_columns_median": statistics.median(host_status)}

try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:  # noqa: BLE001
    q = f"nvidia-smi unavailable: {e}"
res["card"] = torch.cuda.get_device_name(0)
res["nvidia_smi_name_power_limit"] = q
text = json.dumps(res, indent=1)
print(text)
if a.out:
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        f.write(text)
