"""Hold in flight (am_sweep_set_hold_in_flight) against the hold off: the config-2 population (10 M records by default).

Part 1, device-resident ticks (am_sweep_tick_device, as in bench.py's timed loop), alternated in every round at an
on-minute T and an off-minute T:
  off        the hold off (the plain variants);
  on_clean   the hold on from a clean state: every due record is submitted (and its since stored);
  on_held    the hold on, the same tick again: every due record is already held.
Kernel time: the sweep kernel between CUDA events (am_sweep_set_profiling, a pass of its own: the extra events break the
programmatic launch chain).  Step time: CUDA events around the whole call with profiling off.

Part 2, a controller loop: 120 am_sweep_tick_view calls at consecutive seconds; the workflows the loop submitted at
t - 20 post Succeeded before the tick at t.  Reports list entries per tick and the host time of each call (drain +
kernels + one synchronisation), hold off against hold on, alternated.

AMSWEEP_LIB may point at another build of the same ABI, to compare two forms of the kernel in one session.  Prints one
JSON object, with the card's name, power limit and the library it ran."""
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
ap.add_argument("--loop", type=int, default=120)
ap.add_argument("--loop-reps", type=int, default=2)
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
CASES = [(m, c) for m in ("on_minute", "off_minute") for c in ("off", "on_clean", "on_held")]
kern = {k: [] for k in CASES}
step = {k: [] for k in CASES}
emitted = {}

with am.Sweep(capacity=a.n) as s:
    s.load_range(0, cols)

    def tick(T):
        s.tick_device(T, 0, d_idx.data_ptr(), d_act.data_ptr(), a.n, d_cnt.data_ptr(), d_st.data_ptr(), stream.cuda_stream)

    def timed(T, key, profiled):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        tick(T)
        e1.record(stream)
        torch.cuda.synchronize()
        if profiled:
            kern[key].append(s.last_profile()[0])
        else:
            step[key].append(e0.elapsed_time(e1))
            emitted[key] = int(d_st[1].item())

    for profiled in (True, False):
        s.set_profiling(profiled)
        for r in range(a.reps + 3):  # the first three rounds warm up
            for m in ("on_minute", "off_minute"):
                T = T0 + 7 * 86400 * (r + 1) + (0 if m == "on_minute" else 17)
                for c in ("off", "on_clean", "on_held"):
                    if c == "off":
                        s.set_hold_in_flight(False)
                    elif c == "on_clean":
                        s.set_hold_in_flight(True)  # nothing in flight
                        torch.cuda.synchronize()
                    if r < 3:
                        tick(T)
                        torch.cuda.synchronize()
                        continue
                    timed(T, (m, c), profiled)
                s.set_hold_in_flight(False)

    # part 2: the controller loop
    loop = {"off": {"entries": [], "step_ms": []}, "on": {"entries": [], "step_ms": []}}
    for rep in range(a.loop_reps):
        for mode in ("off", "on"):
            s.load_range(0, cols)
            s.set_hold_in_flight(mode == "on")
            subs = {}
            Tl = T0 + 86400 * (100 + rep) - 30  # crosses a minute
            for k in range(a.loop):
                t = Tl + k
                if t - 20 in subs:
                    done = subs.pop(t - 20)
                    if len(done):
                        s.post_result(done, np.full(len(done), am.PHASE_SUCCEEDED, np.uint8))
                t0 = time.perf_counter()
                idx, act, _ = s.tick_view(t)
                dt = (time.perf_counter() - t0) * 1e3
                subs[t] = idx[(act & am.ACT_SUBMIT_HC) != 0].astype(np.uint64)
                loop[mode]["entries"].append(len(idx))
                loop[mode]["step_ms"].append(dt)
    s.set_hold_in_flight(False)

try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:  # noqa: BLE001
    q = f"nvidia-smi unavailable: {e}"
res = {"card": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": q, "n_records": a.n,
       "lib": os.path.basename(am.abi.LIB_PATH), "reps": a.reps, "device_ticks": {}, "controller_loop": {}}
for m, c in CASES:
    res["device_ticks"][f"{m}/{c}"] = {
        "sweep_kernel_ms_median": statistics.median(kern[(m, c)]), "sweep_kernel_ms_min": min(kern[(m, c)]),
        "step_ms_median": statistics.median(step[(m, c)]), "step_ms_min": min(step[(m, c)]),
        "n_emitted_last": emitted[(m, c)]}
for mode, v in loop.items():
    res["controller_loop"][mode] = {"ticks": len(v["entries"]), "entries_per_tick_mean": float(np.mean(v["entries"])),
                                    "entries_per_tick_median": statistics.median(v["entries"]),
                                    "entries_total": int(np.sum(v["entries"])),
                                    "step_ms_median": statistics.median(v["step_ms"]),
                                    "step_ms_p90": float(np.percentile(v["step_ms"], 90))}
out = json.dumps(res, indent=1)
print(out)
if a.out:
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        f.write(out)
