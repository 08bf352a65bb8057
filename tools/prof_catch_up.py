"""Catch-up ticks (AM_SWEEP_CATCH_UP) beside plain on-minute ticks: the config-2 population (10 M records by
default), device-resident ticks (am_sweep_tick_device, as in bench.py's timed loop), windows of 60 s, 3 600 s and
86 400 s and the plain tick alternated in one run.  Kernel time: the sweep kernel between CUDA events
(am_sweep_set_profiling, a pass of its own: the extra events break the programmatic launch chain).  Step time:
CUDA events around the whole call (drain + window upload + sweep + scan + expand + publish) with profiling off.
Prints one JSON object, with the card's name and power limit."""
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
ap.add_argument("--reps", type=int, default=30)
ap.add_argument("--out", default="")
a = ap.parse_args()
am = importlib.import_module("active-monitor_b200")
import torch  # noqa: E402

T0 = amgen.T0_MON_0915  # on the minute
cols = amgen.fill(2, 2, 0, a.n, T0, am.load().am_healthcheck_classify)
kind = cols["flags"] & np.uint32(am.KIND_MASK)
cron = kind == am.KIND_CRON_SPEC
seg = np.zeros((a.n + 127) // 128 * 128, dtype=bool)
seg[: a.n] = cron
cron_warps = int(seg.reshape(-1, 128).any(axis=1).sum())
bytes_window = a.n * 16 + cron_warps * 128 * 40  # flags + ras + finishedAt; five masks in warps with a CRON_SPEC record

dev = torch.device("cuda", 0)
d_idx = torch.empty(a.n, dtype=torch.int32, device=dev)
d_act = torch.empty(a.n, dtype=torch.uint8, device=dev)
d_cnt = torch.zeros(1, dtype=torch.int32, device=dev)
d_st = torch.zeros(16, dtype=torch.int64, device=dev)
stream = torch.cuda.current_stream()
VARIANTS = [("plain_on_minute", 0), ("catch_up_60s", 60), ("catch_up_3600s", 3600), ("catch_up_86400s", 86400)]
kern = {v: [] for v, _ in VARIANTS}
step = {v: [] for v, _ in VARIANTS}
emitted = {}

with am.Sweep(capacity=a.n) as s:
    s.load_range(0, cols)

    def tick(T, mode):
        s.tick_device(T, mode, d_idx.data_ptr(), d_act.data_ptr(), a.n, d_cnt.data_ptr(), d_st.data_ptr(),
                      stream.cuda_stream)

    for profiled in (True, False):
        s.set_profiling(profiled)
        for r in range(a.reps + 3):  # the first three rounds warm up
            T = T0 + 7 * 86400 * (r + 1) + (2 if profiled else 0) * 86400
            for name, w in VARIANTS:
                T += 3 * 86400
                tick(T - (w or 61), 0)  # the previous tick: P = T - w (an off-window second for the plain one)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                tick(T, am.SWEEP_CATCH_UP if w else 0)
                e1.record(stream)
                torch.cuda.synchronize()
                if r < 3:
                    continue
                if profiled:
                    kern[name].append(s.last_profile()[0])
                else:
                    step[name].append(e0.elapsed_time(e1))
                    emitted[name] = int(d_st[1].item())

try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:  # noqa: BLE001
    q = f"nvidia-smi unavailable: {e}"
res = {"card": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": q, "n_records": a.n,
       "cron_spec_share": float(cron.mean()), "warps_with_cron_spec_share": cron_warps / (seg.size // 128),
       "window_variant_bytes_read": bytes_window, "window_variant_bytes_per_record": bytes_window / a.n,
       "reps": a.reps, "variants": {}}
for name, _ in VARIANTS:
    km, sm_ = statistics.median(kern[name]), statistics.median(step[name])
    res["variants"][name] = {"sweep_kernel_ms_median": km, "sweep_kernel_ms_min": min(kern[name]),
                             "step_ms_median": sm_, "step_ms_min": min(step[name]), "n_emitted_last": emitted[name]}
    if name != "plain_on_minute":
        res["variants"][name]["window_bytes_per_s_at_median"] = bytes_window / (km * 1e-3)
out = json.dumps(res, indent=1)
print(out)
if a.out:
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        f.write(out)
