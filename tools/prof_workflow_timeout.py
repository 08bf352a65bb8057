"""Workflow timeouts (am_record_t.wf_timeout with the hold in flight) against the hold alone: the config-2 population
(10 M records by default), two handles loaded alike — `hold` (every wf_timeout 0: no timeout state) and `timeouts`
(a wf_timeout on every record) — alternated in every round.

Part 1, device-resident ticks (am_sweep_tick_device, as in bench.py's timed loop), with wf_timeout = 10^6 (nothing
expires), at an on-minute and an off-minute T:
  clean  the hold turned on again: every due record is submitted (since and, with timeouts, its deadline stored);
  held   the same tick again: every due record is held; the expiry pass finds no segment due.
Kernel times: sweep_tick_kernel between CUDA events (am_sweep_set_profiling, a pass of its own); the expiry pass
(expire_runs_kernel) from torch.profiler over the timed pass.  Step time: CUDA events around the whole call.

Part 2, a controller loop: am_sweep_tick_view at consecutive seconds; 90 % of the workflows submitted at t - 20 post
Succeeded before the tick at t, the rest never post.  `timeouts` has wf_timeout = 60: those time out.  Reports list
entries, timed-out runs per tick and the host time of each call (drain + kernels + one synchronisation).

Part 3, the burst: wf_timeout = 30 on every record, the hold turned on again, a tick at T submits every due record,
then the tick at T + 30 times every one of them out at once (the hold alone: the same two ticks).

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
ap.add_argument("--loop", type=int, default=120)
ap.add_argument("--out", default="")
a = ap.parse_args()
am = importlib.import_module("active-monitor_b200")
import torch  # noqa: E402

T0 = amgen.T0_MON_0915  # on the minute
cols = amgen.fill(2, 2, 0, a.n, T0, am.load().am_healthcheck_classify)
recs = am.columns_to_records(cols)
ALL = np.arange(a.n, dtype=np.uint64)

dev = torch.device("cuda", 0)
d_idx = torch.empty(a.n, dtype=torch.int32, device=dev)
d_act = torch.empty(a.n, dtype=torch.uint8, device=dev)
d_cnt = torch.zeros(1, dtype=torch.int32, device=dev)
d_st = torch.zeros(16, dtype=torch.int64, device=dev)
stream = torch.cuda.current_stream()
HANDLES = ("hold", "timeouts")


def set_w(s, w):
    """every record upserted again with wf_timeout w (the columns as loaded)"""
    s.load_range(0, cols)
    r = recs.copy()
    r["wf_timeout"] = w
    s.upsert(ALL, r)


def tick(s, T):
    s.tick_device(T, 0, d_idx.data_ptr(), d_act.data_ptr(), a.n, d_cnt.data_ptr(), d_st.data_ptr(), stream.cuda_stream)


def kernel_ms(prof, name):
    out = []
    for e in prof.events():
        if name in e.name and str(getattr(e, "device_type", "")).endswith("CUDA"):
            t = getattr(e, "device_time", None) or getattr(e, "cuda_time", 0)
            out.append(t / 1e3)
    return out


res = {"n_records": a.n, "reps": a.reps, "lib": None, "device_ticks": {}, "controller_loop": {}, "burst": {}}
with am.Sweep(capacity=a.n) as h, am.Sweep(capacity=a.n) as x:
    res["lib"] = os.path.basename(am.abi.LIB_PATH)
    sw = {"hold": h, "timeouts": x}
    for s in (h, x):
        s.set_hold_in_flight(True)
    set_w(h, 0)
    set_w(x, 1_000_000)
    torch.cuda.synchronize()

    # ---- part 1
    CASES = [(m, c, k) for m in ("on_minute", "off_minute") for c in ("clean", "held") for k in HANDLES]
    kern = {c: [] for c in CASES}
    step = {c: [] for c in CASES}
    emitted = {}
    expire = {}
    for profiled in (True, False):
        for s in (h, x):
            s.set_profiling(profiled)
        prof = None
        if not profiled:
            prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
            prof.__enter__()
        for r in range(a.reps + 3):  # the first three rounds warm up
            for m in ("on_minute", "off_minute"):
                T = T0 + 7 * 86400 * (r + 1) + (0 if m == "on_minute" else 17)
                for k in HANDLES:
                    s = sw[k]
                    for c in ("clean", "held"):
                        if c == "clean":
                            s.set_hold_in_flight(False)
                            s.set_hold_in_flight(True)
                        torch.cuda.synchronize()
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(stream)
                        tick(s, T)
                        e1.record(stream)
                        torch.cuda.synchronize()
                        if r < 3:
                            continue
                        if profiled:
                            kern[(m, c, k)].append(s.last_profile()[0])
                        else:
                            step[(m, c, k)].append(e0.elapsed_time(e1))
                            emitted[(m, c, k)] = int(d_st[1].item())
        if prof is not None:
            prof.__exit__(None, None, None)
            ms = kernel_ms(prof, "expire_runs_kernel")
            expire = {"launches": len(ms), "ms_median": statistics.median(ms) if ms else None,
                      "ms_max": max(ms) if ms else None}
    for s in (h, x):
        s.set_profiling(False)
    for m, c, k in CASES:
        res["device_ticks"][f"{m}/{c}/{k}"] = {
            "sweep_kernel_ms_median": statistics.median(kern[(m, c, k)]),
            "step_ms_median": statistics.median(step[(m, c, k)]), "step_ms_min": min(step[(m, c, k)]),
            "n_emitted_last": emitted[(m, c, k)]}
    res["device_ticks"]["expire_runs_kernel_nothing_due"] = expire

    # ---- part 2
    set_w(x, 60)
    rng = np.random.default_rng(7)
    loop = {k: {"entries": [], "timed_out": [], "step_ms": []} for k in HANDLES}
    for k in HANDLES:
        s = sw[k]
        s.set_hold_in_flight(False)
        s.set_hold_in_flight(True)
        subs = {}
        Tl = T0 + 86400 * 100 - 30  # crosses a minute
        for j in range(a.loop):
            t = Tl + j
            if t - 20 in subs:
                done = subs.pop(t - 20)
                done = done[rng.random(len(done)) < 0.9]
                if len(done):
                    s.post_result(done, np.full(len(done), am.PHASE_SUCCEEDED, np.uint8))
            t0 = time.perf_counter()
            idx, act, _ = s.tick_view(t)
            dt = (time.perf_counter() - t0) * 1e3
            subs[t] = idx[(act & am.ACT_SUBMIT_HC) != 0].astype(np.uint64)
            loop[k]["entries"].append(len(idx))
            loop[k]["timed_out"].append(len(s.last_timed_out()[0]))
            loop[k]["step_ms"].append(dt)
    for k, v in loop.items():
        res["controller_loop"][k] = {"ticks": len(v["entries"]), "entries_per_tick_mean": float(np.mean(v["entries"])),
                                     "timed_out_total": int(np.sum(v["timed_out"])),
                                     "step_ms_median": statistics.median(v["step_ms"]),
                                     "step_ms_p90": float(np.percentile(v["step_ms"], 90))}

    # ---- part 3
    set_w(x, 30)
    for k in HANDLES:
        s = sw[k]
        s.set_hold_in_flight(False)
        s.set_hold_in_flight(True)
        Tb = T0 + 86400 * 200
        tick(s, Tb)
        torch.cuda.synchronize()
        submitted = int(d_st[2].item())
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            e0.record(stream)
            tick(s, Tb + 30)
            e1.record(stream)
            torch.cuda.synchronize()
        t0 = time.perf_counter()
        n_to = len(s.last_timed_out()[0])
        read_ms = (time.perf_counter() - t0) * 1e3
        ms = kernel_ms(prof, "expire_runs_kernel")
        res["burst"][k] = {"submitted_at_T": submitted, "timed_out_at_T_plus_30": n_to, "step_ms": e0.elapsed_time(e1),
                           "expire_runs_kernel_ms": ms[0] if ms else None, "n_result_fail": int(d_st[11].item()),
                           "last_timed_out_host_ms": read_ms}

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
