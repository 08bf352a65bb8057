"""tests/test_on_demand_adversarial_gpu.py on the CPU emulator: the library compiled for tests/emu (same kernel and host
sources) behind the real C-ABI, in a child process, as tests/test_workflow_timeout_emulator.py does for the workflow
timeouts.  The 10 M-record next_due case stays on the GPU."""
import os
import subprocess
import sys

from conftest import ROOT

EMU = os.path.join(ROOT, "tests", "emu")


def test_on_demand_adversarial_suite_on_the_emulated_library():
    sys.path.insert(0, EMU)
    import emu_sweep
    env = dict(os.environ, AMSWEEP_LIB=emu_sweep.build())
    out = subprocess.run([sys.executable, "-m", "pytest", "tests/test_on_demand_adversarial_gpu.py", "-m", "gpu", "-q",
                          "-x", "-p", "no:cacheprovider", "-k", "not 10m"], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=1800)
    tail = out.stdout[-3000:] + out.stderr[-2000:]
    assert out.returncode == 0, tail
    last = out.stdout.strip().splitlines()[-1]
    assert " passed" in last and " failed" not in last and "error" not in last and "skipped" not in last, tail
    assert "1 xfailed" in last, tail  # the half-hour daylight-saving gap
    assert int(last.split(" passed")[0].split()[-1]) >= 249, tail
