"""The remedy hold (am_sweep_set_hold_remedy) against the hold with workflow timeouts alone: the config-3 population
(remedy actions; 10 M records by default), two handles loaded alike with the hold on and a wf_timeout of 10^6 on every
record (nothing expires) — `hold` (remedy hold off) and `remedy` (remedy hold on) — alternated in every round.

Part 1, device-resident ticks (am_sweep_tick_device, as in bench.py's timed loop), per round on each handle: both holds
turned on again, the tick at T submits every due record, then
  sparse  1 % of them post Failed (applied by the drain's result kernel), timed tick at T + 1;
  dense   50 % of them post Failed (more than an eighth of the records: applied inside the sweep), timed tick at T + 2;
  held    the tick at T + 3 with nothing posted: every submitted record is held.
Kernel times: sweep_tick_kernel between CUDA events (am_sweep_set_profiling, a pass of its own).  Step time: CUDA events
around the whole call, in the other pass.

Part 2, a controller loop: am_sweep_tick_view at consecutive seconds; of the workflows submitted at t - 20, 70 % post
Succeeded and 30 % Failed before the tick at t; every remedy started at t - 40 posts Succeeded before the tick at t.
Reports list entries, RUN_REMEDY entries per tick and the host time of each call.

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
ap.add_argument("--reps", type=int, default=15)
ap.add_argument("--loop", type=int, default=120)
ap.add_argument("--out", default="")
a = ap.parse_args()
am = importlib.import_module("active-monitor_b200")
import torch  # noqa: E402

T0 = amgen.T0_MON_0915  # on the minute
cols = amgen.fill(3, 3, 0, a.n, T0, am.load().am_healthcheck_classify)
recs = am.columns_to_records(cols)
recs["wf_timeout"] = 1_000_000
ALL = np.arange(a.n, dtype=np.uint64)

dev = torch.device("cuda", 0)
d_idx = torch.empty(a.n, dtype=torch.int32, device=dev)
d_act = torch.empty(a.n, dtype=torch.uint8, device=dev)
d_cnt = torch.zeros(1, dtype=torch.int32, device=dev)
d_st = torch.zeros(16, dtype=torch.int64, device=dev)
stream = torch.cuda.current_stream()
HANDLES = ("hold", "remedy")
PARTS = ("sparse", "dense", "held")


def reset(s, k):
    s.set_hold_in_flight(False)
    s.set_hold_in_flight(True)
    if k == "remedy":
        s.set_hold_remedy(True)


def tick(s, T):
    s.tick_device(T, 0, d_idx.data_ptr(), d_act.data_ptr(), a.n, d_cnt.data_ptr(), d_st.data_ptr(), stream.cuda_stream)


def submitted():
    n = int(d_cnt.item())
    act = d_act[:n].cpu().numpy()
    return d_idx[:n].cpu().numpy().astype(np.uint64)[(act & am.ACT_SUBMIT_HC) != 0]


res = {"n_records": a.n, "reps": a.reps, "device_ticks": {}, "controller_loop": {}}
with am.Sweep(capacity=a.n) as h, am.Sweep(capacity=a.n) as x:
    sw = {"hold": h, "remedy": x}
    for s in (h, x):
        s.load_range(0, cols)
        s.set_hold_in_flight(True)
        s.upsert(ALL, recs)
    rng = np.random.default_rng(3)

    # ---- part 1
    kern = {(p, k): [] for p in PARTS for k in HANDLES}
    step = {(p, k): [] for p in PARTS for k in HANDLES}
    runs = {}
    for profiled in (True, False):
        for r in range(a.reps + 2):  # the first two rounds warm up
            T = T0 + 7 * 86400 * (r + 1)
            for k in HANDLES:
                s = sw[k]
                s.set_profiling(profiled)
                reset(s, k)
                tick(s, T)
                sub = submitted()
                for j, p in enumerate(PARTS):
                    frac = {"sparse": 0.01, "dense": 0.5, "held": 0.0}[p]
                    sl = sub[rng.random(len(sub)) < frac]
                    if len(sl):
                        s.post_result(sl, np.full(len(sl), am.PHASE_FAILED, np.uint8))
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    tick(s, T + 1 + j)
                    e1.record(stream)
                    torch.cuda.synchronize()
                    if r < 2:
                        continue
                    if profiled:
                        kern[(p, k)].append(s.last_profile()[0])
                    else:
                        step[(p, k)].append(e0.elapsed_time(e1))
                        runs[(p, k)] = {"posted_failed": int(len(sl)), "n_emitted": int(d_st[1].item()),
                                        "n_submit_hc": int(d_st[2].item()), "n_run_remedy": int(d_st[3].item())}
                s.set_profiling(False)
    for p in PARTS:
        for k in HANDLES:
            res["device_ticks"][f"{p}/{k}"] = {"sweep_kernel_ms_median": statistics.median(kern[(p, k)]),
                                               "step_ms_median": statistics.median(step[(p, k)]), **runs[(p, k)]}

    # ---- part 2
    for k in HANDLES:
        s = sw[k]
        reset(s, k)
        subs, rems = {}, {}
        out = {"entries": [], "run_remedy": [], "step_ms": []}
        Tl = T0 + 86400 * 100 - 30  # crosses a minute
        for j in range(a.loop):
            t = Tl + j
            if t - 20 in subs:
                done = subs.pop(t - 20)
                ph = np.where(rng.random(len(done)) < 0.7, am.PHASE_SUCCEEDED, am.PHASE_FAILED).astype(np.uint8)
                if len(done):
                    s.post_result(done, ph)
            if t - 40 in rems and len(rems[t - 40]):
                r_done = rems.pop(t - 40)
                s.post_result(r_done, np.zeros(len(r_done), np.uint8), np.full(len(r_done), am.PHASE_SUCCEEDED, np.uint8))
            t0 = time.perf_counter()
            idx, act, _ = s.tick_view(t)
            dt = (time.perf_counter() - t0) * 1e3
            subs[t] = idx[(act & am.ACT_SUBMIT_HC) != 0].astype(np.uint64)
            rems[t] = idx[(act & am.ACT_RUN_REMEDY) != 0].astype(np.uint64)
            out["entries"].append(len(idx))
            out["run_remedy"].append(len(rems[t]))
            out["step_ms"].append(dt)
        res["controller_loop"][k] = {"ticks": a.loop, "entries_per_tick_mean": float(np.mean(out["entries"])),
                                     "run_remedy_total": int(np.sum(out["run_remedy"])),
                                     "step_ms_median": statistics.median(out["step_ms"]),
                                     "step_ms_p90": float(np.percentile(out["step_ms"], 90))}

try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:  # noqa: BLE001
    q = f"nvidia-smi unavailable: {e}"
res["card"] = torch.cuda.get_device_name(0)
res["nvidia_smi_name_power_limit"] = q
out = json.dumps(res, indent=1)
print(out)
if a.out:
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        f.write(out)
