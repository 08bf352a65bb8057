"""The NVLink tick exchange (csrc/gather.cu + gather_kernels.cuh + the list rebuild of
sweep_kernels.cuh) on a CPU emulation of the CUDA execution model (tests/emu): ranks are OS
threads, a CTA's threads are fibers, `__syncthreads` and the warp collectives are rendezvous
points, system-scope acquire/release are std atomics.

The SAME sources the GPU runs are compiled for the host; every rank sweeps its index-range shard
of ONE population and exchanges several ticks back to back (no host barrier, as on the stream);
every rank's global list, counts, shard statistics and final columns must equal the UNSHARDED
oracle.  This covers the N>1 path's index arithmetic, slot layout and epoch / ticket / done-flag
protocol without a GPU; it does not cover the GPU memory model or performance — the `-m gpu`
tests in tests/test_multi_gpu.py do, on 2 / 4 / 8 H100s.
"""
import os
import subprocess
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402


def _run(args, env=None, timeout=900):
    return emu_sweep.run_script("run_gather_ranks.py", args, env, timeout)


# world, idx_bytes, records in total, ticks, population
CASES = [
    (2, 4, 40_000, 4, 3),      # config 3: dense exceptions (remedy actions)
    (2, 8, 40_000, 4, 2),      # config 2: sparse exceptions, u64 indices
    (3, 8, 30_011, 4, 3),      # ragged shard sizes, partial last group and tile
    (4, 4, 36_000, 4, 2),
    (8, 4, 65_536, 3, 3),      # exactly one 8192-record group per rank
    (8, 8, 9_000, 3, 2),       # shards smaller than a group, more CTAs than tiles
    (5, 4, 5, 2, 2),           # one record per rank
    (2, 4, 600_000, 2, 2),     # 37 groups per rank
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "w{}_b{}_n{}_t{}_c{}".format(*c))
def test_exchanged_ticks_equal_the_unsharded_oracle(case):
    _run(["tick"] + list(case))


@pytest.mark.parametrize("case", [(2, 4, 40_000, 4, 3), (3, 8, 30_011, 4, 2), (8, 4, 65_536, 3, 3), (5, 4, 5, 2, 2)],
                         ids=lambda c: "w{}_b{}_n{}_t{}_c{}".format(*c))
def test_whole_step_in_one_call_returns_the_ranks_own_part_as_local_slots(case):
    """am_gather_bind + am_gather_tick_view: tick_shard + exchange + extraction of the rank's own part of the
    global list into pinned host memory, one synchronisation; the global list, the shard statistics and the view
    must all equal the oracle's."""
    _run(["tick"] + list(case), env={"EMU_TICK_VIEW": "1"})


def test_whole_step_reports_an_absent_peer_as_an_error():
    out = _run(["tick", 3, 4, 30_000, 3], env={"EMU_ABSENT_RANK": "1", "AMSWEEP_PUSH_TIMEOUT_MS": "300",
                                                         "EMU_TICK_VIEW": "1"}, timeout=120)
    assert "watchdog" in out


@pytest.mark.parametrize("ctas", [1, 3, 40])
def test_any_push_grid_size(ctas):
    _run(["tick", 3, 4, 50_000, 3, 3], env={"AMSWEEP_PUSH_CTAS": str(ctas)})


def test_protocol_survives_skew_between_ranks():
    """EMU_JITTER: random pauses at launches and system-scope stores let ranks drift apart by whole
    kernels over 25 back-to-back ticks; the epoch / done-flag / two-slot-set protocol must still
    deliver the oracle's list on every rank."""
    _run(["tick", 4, 4, 48_000, 25, 2], env={"EMU_JITTER": "1"})


def test_a_fast_rank_may_finish_its_next_push_before_a_slow_one_has_seen_this_one():
    """Tiny shards, 8 ranks, 40 ticks, skew: a rank regularly raises done(e+1) while a peer still waits
    for its done(e) — the wait must accept ">= e" (round-2 bug found here: waiting for "== e" let the
    slow rank run into the watchdog)."""
    _run(["tick", 8, 8, 9_000, 40, 2], env={"EMU_JITTER": "1", "AMSWEEP_PUSH_TIMEOUT_MS": "20000"})
    _run(["tick", 8, 4, 9_000, 40, 3])


def test_watchdog_gives_up_on_an_absent_peer():
    """The device-side wait for the peers' done flags is bounded (AMSWEEP_PUSH_TIMEOUT_MS): a rank that
    never exchanges makes the others report 0xFFFFFFFF in out_counts[world] instead of hanging the GPU."""
    out = _run(["tick", 3, 4, 30_000, 3], env={"EMU_ABSENT_RANK": "1", "AMSWEEP_PUSH_TIMEOUT_MS": "300"},
               timeout=120)
    assert "watchdog" in out


@pytest.mark.parametrize("world,idx_bytes,records", [(2, 4, 20_000), (3, 8, 30_011), (8, 4, 9_000)])
def test_round1_plain_list_format_still_equals_the_concatenation(world, idx_bytes, records):
    _run(["plain", world, idx_bytes, records, 5])


def test_flag_protocol_orders_every_cross_rank_access_under_threadsanitizer(tmp_path):
    """tests/emu/tsan_exchange.cpp: the library's own sources on the emulator, built with
    -fsanitize=thread (the emulator tells TSan about its fibers; every fiber switch synchronises, so
    only accesses of DIFFERENT ranks can race).  Three ranks as threads tick and exchange back to back.
    System-scope release/acquire are atomics there, everything else — peer payload stores, slot reads
    by the list rebuild — plain memory accesses: a report would mean some cross-rank data is not
    ordered by the done-flag protocol."""
    exe = emu_sweep.build_tsan("tsan_exchange.cpp", str(tmp_path / "tsan_exchange.bin"))
    out = subprocess.run([exe], capture_output=True, text=True, timeout=900,
                         env=dict(os.environ, TSAN_OPTIONS="halt_on_error=0 exitcode=66"))
    assert "ThreadSanitizer" not in out.stderr, out.stderr[-3000:]
    assert out.returncode == 0 and out.stdout.startswith("ok"), out.stdout + out.stderr[-2000:]
