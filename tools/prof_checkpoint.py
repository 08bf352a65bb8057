"""Checkpoint and restore of a sweep handle at BASELINE config 5's 10 M records in the configuration INTEGRATION.md §3
recommends (the hold in flight, the remedy hold, workflow timeouts on a tenth of the slots, status changes with
details), after a simulated hour so that runs are in flight.  Measured, alternating the paths, each repeated:

  guard_ms       the tick guard held by am_sweep_checkpoint (drain + the packing pass): a second thread ticks the
                 handle in a loop during the call; the span from its first to its last AM_E_BUSY answer
  checkpoint_ms  the whole am_sweep_checkpoint call (the pass, then the copy of the blob into pageable host memory)
  restore_ms     the whole am_sweep_restore call into a fresh handle with the same switches
  read_load_ms   am_sweep_read of the sixteen columns + am_sweep_load_range of them (the path before checkpoints)
  memcpy_d2h_ms / memcpy_h2d_ms   a plain cudaMemcpy of the blob's byte count between pinned host memory and HBM

The card's name and power limit are read in the same run.  Prints one
JSON object."""
import argparse
import importlib
import json
import os
import statistics
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tools", "amgen")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import run_sim  # noqa: E402


def handle(am, cols, sl, recs):
    n = len(cols["flags"])
    s = am.Sweep(capacity=n)
    s.load_range(0, cols)
    s.set_hold_in_flight(True)
    s.set_hold_remedy(True)
    s.set_track_changes(True)
    s.set_change_details(True)
    s.upsert(sl, recs)
    return s


def retry_busy(am, call):
    """`call` again while it meets a tick in progress (AM_E_BUSY)"""
    while True:
        try:
            return call()
        except am.AmError as e:
            if e.code != am.AM_E_BUSY:
                raise


def busy_span(am, s, T, call):
    """run `call` while another thread ticks s at T (AM_E_BUSY answers counted): (result, ms the ticks were refused)"""
    stop, spans = threading.Event(), []
    idx, act = np.empty(s.capacity, np.uint64), np.empty(s.capacity, np.uint32)

    def ticker():
        first = last = None
        while not stop.is_set():
            t0 = time.perf_counter()
            try:
                s.tick(T, buffers=(idx, act))
            except am.AmError as e:
                if e.code != am.AM_E_BUSY:
                    raise
                first = t0 if first is None else first
                last = time.perf_counter()
        spans.append(0.0 if first is None else (last - first) * 1e3)

    th = threading.Thread(target=ticker)
    th.start()
    time.sleep(0.05)
    try:
        out = call()
    finally:
        stop.set()
        th.join()
    return out, spans[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--repeat", type=int, default=5)
    a = ap.parse_args()
    am = importlib.import_module("active-monitor_b200")
    import torch
    cols, sl, recs = run_sim.population(am, a.n, run_sim.SEED)
    s = handle(am, cols, sl, recs)
    T0 = run_sim.amgen.T0_DAY_START
    s.simulate(T0, 3600, am.SWEEP_BLOCKED, run_sim.SEED, run_sim.PARAMS)
    T = T0 + 3600
    blob = s.checkpoint(0, a.n)
    info = am.checkpoint_info(blob)
    nbytes = info["bytes"]
    pinned = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    dev = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    out = {"workload": f"config 5: {a.n} records, a simulated hour (hold in flight, remedy hold, a tenth with workflow "
                       f"timeouts, status changes with details), then a checkpoint of every slot",
           "card": run_sim.card(), "blob_bytes": nbytes, "bytes_per_slot": nbytes / a.n, "switches": info["switches"]}
    times = {k: [] for k in ("checkpoint_ms", "guard_ms", "restore_ms", "read_load_ms", "memcpy_d2h_ms",
                             "memcpy_h2d_ms")}
    for _ in range(a.repeat):
        # the checkpoint: the whole call, and the span a concurrent ticker is refused
        t0 = time.perf_counter()
        b = s.checkpoint(0, a.n)
        times["checkpoint_ms"].append((time.perf_counter() - t0) * 1e3)
        _, busy = busy_span(am, s, T, lambda: retry_busy(am, lambda: s.checkpoint(0, a.n)))
        times["guard_ms"].append(busy)
        # the restore into a fresh handle with the same switches
        t = am.Sweep(capacity=a.n)
        t.set_hold_in_flight(True)
        t.set_hold_remedy(True)
        t.set_track_changes(True)
        t.set_change_details(True)
        t0 = time.perf_counter()
        t.restore(b)
        times["restore_ms"].append((time.perf_counter() - t0) * 1e3)
        t.close()
        del b
        # the path before checkpoints: read the sixteen columns, load them
        u = am.Sweep(capacity=a.n)
        t0 = time.perf_counter()
        c = s.read_range(0, a.n)
        u.load_range(0, c)
        times["read_load_ms"].append((time.perf_counter() - t0) * 1e3)
        u.close()
        del c
        # plain pinned copies of the blob's byte count
        for k, (dst, src) in (("memcpy_d2h_ms", (pinned, dev)), ("memcpy_h2d_ms", (dev, pinned))):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            dst.copy_(src)
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3)
    out["ms"] = {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in times.items()}
    out["card_after"] = run_sim.card()
    s.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
