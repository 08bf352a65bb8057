"""Checkpoints, delta chains and restores against concurrent calls on the CPU tier.

ThreadSanitizer: tests/emu/tsan_checkpoint.cpp runs four stagers (upsert, remove, post_result, update_spec), a ticker,
a checkpointer (two chains, deltas with the AM_E_NOSPACE path, full checkpoints, am_checkpoint_delta_info), a querier and
a restorer on one handle with the hold, details and a finite submit budget on, built with the library's own sources
on the emulator.  It passes with exit status 0 and no TSan report.

The thread cases of tests/test_checkpoint_threads_gpu.py (a ticker, a poster, a checkpointer and a querier; a restore
into a ticking handle; am_sweep_restore_delta after a tick of every entry point; zero padding in blobs) on the
emulated library at a small size, in a child process.  Its stream cases need a GPU: the emulated library completes
every call before it returns."""
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402


def test_checkpoint_threads_under_thread_sanitizer():
    with tempfile.TemporaryDirectory() as d:
        exe = emu_sweep.build_tsan("tsan_checkpoint.cpp", os.path.join(d, "tsan_checkpoint"))
        r = subprocess.run([exe], capture_output=True, text=True, timeout=900,
                           env=dict(os.environ, TSAN_OPTIONS="halt_on_error=1 exitcode=66"))
    assert r.returncode == 0 and "WARNING: ThreadSanitizer" not in r.stderr, r.stdout[-2000:] + r.stderr[-6000:]
    assert r.stdout.startswith("ok"), r.stdout[-2000:]


def test_checkpoint_thread_cases_on_the_emulated_library():
    got = emu_sweep.run_suite("tests/test_checkpoint_threads_gpu.py",
                              k="ticker_poster or ticking_handle or refused_after_a_tick or padding")
    assert got["passed"] == 10, got
