"""tests/test_change_details_gpu.py on the CPU emulator: the library compiled for tests/emu (same kernel and host sources)
behind the real C-ABI, in a child process, as tests/test_status_changes_emulator.py does for the status changes.  The
10 M-record comparison stays on the GPU."""
import os
import subprocess
import sys

import pytest

from conftest import ROOT

EMU = os.path.join(ROOT, "tests", "emu")


def test_change_details_suite_on_the_emulated_library():
    sys.path.insert(0, EMU)
    import emu_sweep
    env = dict(os.environ, AMSWEEP_LIB=emu_sweep.build())
    out = subprocess.run([sys.executable, "-m", "pytest", "tests/test_change_details_gpu.py", "-m", "gpu", "-q", "-x",
                          "-p", "no:cacheprovider", "-k", "not full_size"], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=1800)
    tail = out.stdout[-3000:] + out.stderr[-2000:]
    assert out.returncode == 0, tail
    last = out.stdout.strip().splitlines()[-1]
    assert " passed" in last and "failed" not in last and "skipped" not in last, tail
    assert int(last.split(" passed")[0].split()[-1]) >= 80, tail


@pytest.mark.parametrize("case", [(2, 4, 20_000, 22), (3, 8, 30_011, 3)], ids=lambda c: "w{}_b{}_n{}_c{}".format(*c))
def test_each_shard_reports_its_own_details_through_am_gather_tick_view(case):
    """tests/emu/run_gather_change_details.py: every rank's details against the oracle of the unsharded population"""
    sys.path.insert(0, EMU)
    import emu_sweep
    out = subprocess.run([sys.executable, os.path.join(EMU, "run_gather_change_details.py")] + [str(a) for a in case],
                         cwd=ROOT, env=dict(os.environ, AMSWEEP_LIB=emu_sweep.build()), capture_output=True, text=True,
                         timeout=900)
    assert out.returncode == 0 and out.stdout.strip().startswith("ok"), out.stdout[-3000:] + out.stderr[-3000:]
