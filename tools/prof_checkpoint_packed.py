"""Packed checkpoints (format version 2) against raw ones (version 1) at 10 M records after a simulated hour, with the
switches of tools/prof_checkpoint.py (the hold in flight, the remedy hold, workflow timeouts on a tenth of the slots,
status changes with details): BASELINE config 5's population (--config 5), or config 2's (--config 2).  Measured,
the encodings alternated, each repeated:

  bytes                  a full blob raw and packed, and per simulated period of 1, 10 and 60 s a delta's raw and
                         packed length (a packed link's header names the raw length it decodes to)
  checkpoint_ms          the whole Sweep.checkpoint call (pass, encode, copy into pageable host memory)
  restore_ms             the whole Sweep.restore call into a standby with the same switches
  delta_ms               the whole Sweep.checkpoint_delta call; links alternate raw and packed
  restore_delta_ms       the whole Sweep.restore_delta call on a standby that follows the chain
  kernel_ms              the encode's and decode's kernels' device time, from separate torch.profiler runs of one
                         packed 60 s delta with its restore_delta, and of one packed full checkpoint with its restore

The card's name and power limit are read in the same run.  Prints one JSON object."""
import argparse
import importlib
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tools", "amgen")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import run_sim  # noqa: E402
from prof_checkpoint import handle  # noqa: E402
from prof_checkpoint_delta import standby  # noqa: E402

KERNELS = ("ckp_size_kernel", "ckp_write_kernel", "ckp_validate_kernel", "ckp_decode_kernel",
           "checkpoint_pack_kernel", "checkpoint_verify_kernel")


def timed(f):
    t0 = time.perf_counter()
    out = f()
    return out, (time.perf_counter() - t0) * 1e3


def raw_len(blob):
    """the version-1 length a blob stands for (header word 14 of a packed one)"""
    w = np.frombuffer(blob[:128], "<u8")
    return int(w[14]) if int(w[1]) & 0xFFFFFFFF == 2 else len(blob)


def med(v):
    return round(statistics.median(v), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=5, choices=(2, 5))
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--periods", default="1,10,60")
    a = ap.parse_args()
    am = importlib.import_module("active-monitor_b200")
    import torch  # noqa: F401  (CUDA context for the profiler)
    from torch.profiler import ProfilerActivity, profile
    if a.config == 5:
        cols, sl, recs = run_sim.population(am, a.n, run_sim.SEED)
    else:
        cols = run_sim.amgen.fill(2, 2, 0, a.n, run_sim.amgen.T0_DAY_START, am.load().am_healthcheck_classify)
        rng = np.random.default_rng(2)
        sl = np.sort(rng.choice(a.n, a.n // 10, replace=False))
        recs = am.columns_to_records({k: v[sl] for k, v in cols.items()})
        recs["wf_timeout"] = rng.integers(60, 900, len(sl))
    s = handle(am, cols, sl, recs)
    del cols, recs
    T = run_sim.amgen.T0_DAY_START
    s.simulate(T, 3600, am.SWEEP_BLOCKED, run_sim.SEED, run_sim.PARAMS)
    T += 3600
    sb = standby(am, a.n)
    out = {"workload": f"config {a.config}: {a.n} records after a simulated hour (hold in flight, remedy hold, a tenth "
                       f"with workflow timeouts, status changes with details)", "card": run_sim.card()}
    rows = {k: [] for k in ("checkpoint_raw_ms", "checkpoint_packed_ms", "restore_raw_ms", "restore_packed_ms")}
    s.set_checkpoint_packing(True)
    s.checkpoint(0, a.n)  # (the wrapper's kept buffer for packed blobs)
    for r in range(2 * a.repeat):
        packed = r % 2 == 1
        s.set_checkpoint_packing(packed)
        blob, ms = timed(lambda: s.checkpoint(0, a.n))
        rows["checkpoint_packed_ms" if packed else "checkpoint_raw_ms"].append(ms)
        out["full_packed_bytes" if packed else "full_raw_bytes"] = len(blob)
        _, ms = timed(lambda: sb.restore(blob))
        rows["restore_packed_ms" if packed else "restore_raw_ms"].append(ms)
        del blob
    out["full"] = {k: med(v) for k, v in rows.items()}
    out["full"]["ratio"] = round(out["full_packed_bytes"] / out["full_raw_bytes"], 4)
    out["full"]["raw"] = rows
    s.set_checkpoint_packing(False)
    sb.restore(s.checkpoint_chain(0, a.n))
    out["periods"] = {}
    for period in (int(x) for x in a.periods.split(",")):
        rows = {k: [] for k in ("raw_bytes", "packed_bytes", "n_changed", "delta_raw_ms", "delta_packed_ms",
                                "restore_delta_raw_ms", "restore_delta_packed_ms")}
        for r in range(2 * a.repeat):
            packed = r % 2 == 1
            s.set_checkpoint_packing(packed)
            s.simulate(T, period, am.SWEEP_BLOCKED, run_sim.SEED, run_sim.PARAMS)
            T += period
            (d, k), ms = timed(lambda: s.checkpoint_delta())
            kind = "packed" if packed else "raw"
            rows[f"delta_{kind}_ms"].append(ms)
            rows["n_changed"].append(k)
            rows["raw_bytes"].append(raw_len(d))
            if packed:
                rows["packed_bytes"].append(len(d))
            _, ms = timed(lambda: sb.restore_delta(d))
            rows[f"restore_delta_{kind}_ms"].append(ms)
        out["periods"][str(period)] = {k: med(v) for k, v in rows.items()}
        out["periods"][str(period)]["raw"] = rows
    # the kernels' device time, one packed call of each kind under the profiler
    s.set_checkpoint_packing(True)
    s.simulate(T, 60, am.SWEEP_BLOCKED, run_sim.SEED, run_sim.PARAMS)
    T += 60
    out["kernel_ms"] = {}
    for what, calls in (("delta_60s", lambda: sb.restore_delta(s.checkpoint_delta()[0])),  # (first: a full restore
                        ("full", lambda: sb.restore(s.checkpoint(0, a.n)))):             # restarts the link)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            calls()
        out["kernel_ms"][what] = {k: round(sum(e.device_time_total for e in prof.key_averages() if k in e.key) / 1e3, 3)
                                  for k in KERNELS}
    s.set_checkpoint_packing(False)
    out["standby_matches_source"] = sb.checkpoint(0, a.n) == s.checkpoint(0, a.n)
    print(json.dumps(out))
    s.close()
    sb.close()


if __name__ == "__main__":
    main()
