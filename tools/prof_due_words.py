"""The due words of the open-loop tick (due_word, csrc/sweep_kernels.cuh) at config 2, 10 M records by default: two
handles loaded alike, `words` and `columns` (finished_at handed out through am_sweep_column_ptr, so every tick of it
reads ras and finishedAt as the sweep did before the words), alternated in every round.  Kernel times are
sweep_tick_kernel between CUDA events (am_sweep_set_profiling); medians over the rounds.

Part 1, the traffic the sweep shares with its neighbours, on `columns`: its sweep after a tick that wrote the 6 M-entry
list (am_sweep_tick_device; the list's dirty lines leave L2 while the next sweep streams) against its sweep after one
that did not expand (am_sweep_tick_shard).
Part 2, on- and off-minute device ticks of both handles (tick_device at T0 and T0 + 1).
Part 3, the build: a closed-loop tick drops the words, so the next plain tick rebuilds them (DUE = kDueBuild); CUDA
events around that tick against the median plain tick.
Part 4, the e2e loop of bench.py (amgen.e2e_closed_loop: post Succeeded for the previous list, am_sweep_tick_view,
AM_SWEEP_FULL_SCAN) on both handles.

Prints one JSON object, with the card's name and power limit read in the same run."""
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

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=10_000_000)
ap.add_argument("--reps", type=int, default=30)
ap.add_argument("--e2e", type=int, default=100, help="steps of each e2e run")
ap.add_argument("--out", default="")
a = ap.parse_args()
am = importlib.import_module("active-monitor_b200")
import torch  # noqa: E402

T0 = amgen.T0_MON_0915  # on the minute
lib = am.load()
dev = torch.device("cuda", 0)
d_idx = torch.empty(a.n, dtype=torch.int32, device=dev)
d_act = torch.empty(a.n, dtype=torch.uint8, device=dev)
d_cnt = torch.zeros(1, dtype=torch.int32, device=dev)
d_st = torch.zeros(16, dtype=torch.int64, device=dev)
stream = torch.cuda.current_stream()
cols = amgen.fill(2, 2, 0, a.n, T0, lib.am_healthcheck_classify, threads=32)
H = {"words": am.Sweep(capacity=a.n), "columns": am.Sweep(capacity=a.n)}
for s in H.values():
    s.load_range(0, cols)
H["columns"].column_ptr("finished_at")
res = {"n_records": a.n, "reps": a.reps}


def tick_device(s, T, mode=0):
    s.tick_device(T, mode, d_idx.data_ptr(), d_act.data_ptr(), a.n, d_cnt.data_ptr(), d_st.data_ptr(), stream.cuda_stream)


def sweep_ms(s, call):
    """sweep_tick_kernel time of one call of `call` on s"""
    s.set_profiling(True)
    call()
    ms = s.last_profile()[0]
    s.set_profiling(False)
    return ms


def med(v):
    return round(statistics.median(v), 4)


# warm-up: every shape and both handles (the first plain tick of `words` builds its words)
for s in H.values():
    for T in (T0, T0 + 1, T0):
        tick_device(s, T)
    s.tick_shard(T0, 0, stream.cuda_stream)
torch.cuda.synchronize()

# ---- part 1 ----
s = H["columns"]
after = {"tick_device": [], "tick_shard": []}
for _ in range(a.reps):
    tick_device(s, T0)
    after["tick_device"].append(sweep_ms(s, lambda: tick_device(s, T0)))
    s.tick_shard(T0, 0, stream.cuda_stream)
    after["tick_shard"].append(sweep_ms(s, lambda: s.tick_shard(T0, 0, stream.cuda_stream)))
tick_device(s, T0)  # (the shard ticks' statistics are not published: a host-side tick starts the next part clean)
res["part1_columns_sweep_ms_after"] = {k: med(v) for k, v in after.items()}
res["part1_list_write_back_ms"] = round(res["part1_columns_sweep_ms_after"]["tick_device"] -
                                        res["part1_columns_sweep_ms_after"]["tick_shard"], 4)

# ---- part 2 ----
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]


def step_ms(call):
    ev[0].record(stream)
    call()
    ev[1].record(stream)
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1])


part2 = {}
for label, T in (("on_minute", T0), ("off_minute", T0 + 1)):
    sw = {k: [] for k in H}
    st = {k: [] for k in H}
    for _ in range(a.reps):
        for k, s in H.items():
            tick_device(s, T)
            sw[k].append(sweep_ms(s, lambda: tick_device(s, T)))
            st[k].append(step_ms(lambda: tick_device(s, T)))
    part2[label] = {"sweep_ms": {k: med(v) for k, v in sw.items()}, "step_ms": {k: med(v) for k, v in st.items()},
                    "sweep_ms_range": {k: [round(min(v), 4), round(max(v), 4)] for k, v in sw.items()}}
res["part2_device_ticks"] = part2

# ---- part 3 ----
s = H["words"]
plain, rebuilt = [], []
for _ in range(a.reps):
    tick_device(s, T0)
    plain.append(step_ms(lambda: tick_device(s, T0)))
    tick_device(s, T0, am.SWEEP_CLOSED_LOOP)  # drops the words
    rebuilt.append(step_ms(lambda: tick_device(s, T0)))
res["part3_build_extra_ms"] = round(statistics.median(rebuilt) - statistics.median(plain), 4)
res["part3_step_ms"] = {"plain": med(plain), "with_build": med(rebuilt)}

# ---- part 4 ----
e2e = {k: [] for k in H}
for r in range(3):
    for k, s in H.items():
        c = amgen.e2e_closed_loop(lib, s._h, T0 + 1000 + r * (a.e2e + 8), am.SWEEP_FULL_SCAN, 8, a.e2e, a.n)
        e2e[k].append(round(c["seconds"] / a.e2e * 1e3, 4))
res["part4_e2e_ms_per_step"] = {k: {"median": med(v), "runs": v} for k, v in e2e.items()}

try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30).stdout.strip()
except Exception as e:  # noqa: BLE001
    q = f"nvidia-smi unavailable: {e}"
res["nvidia_smi_name_power_limit"] = q
for s in H.values():
    s.close()
out = json.dumps(res)
print(out)
if a.out:
    with open(a.out, "w") as f:
        f.write(out + "\n")
