"""tests/test_call_sequences_gpu.py on the CPU emulator: the library compiled for tests/emu (same kernel and host
sources) behind the real C-ABI, in a child process, as tests/test_catch_up_emulator.py does for catch-up ticks.  The
walks run on smaller handles (SEQ_CAPACITIES); the emulated library completes every call before it returns, so the
walks tick on the handle's own stream only."""
import os
import subprocess
import sys

from conftest import ROOT

EMU = os.path.join(ROOT, "tests", "emu")


def test_call_sequences_on_the_emulated_library():
    sys.path.insert(0, EMU)
    import emu_sweep
    env = dict(os.environ, AMSWEEP_LIB=emu_sweep.build(), SEQ_CAPACITIES="1,257,1025,3001,513,2049")
    out = subprocess.run([sys.executable, "-m", "pytest", "tests/test_call_sequences_gpu.py", "-m", "gpu", "-q", "-x",
                          "-p", "no:cacheprovider"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    tail = out.stdout[-3000:] + out.stderr[-2000:]
    assert out.returncode == 0, tail
    last = out.stdout.strip().splitlines()[-1]
    assert " passed" in last and "failed" not in last and "skipped" not in last, tail
    assert int(last.split(" passed")[0].split()[-1]) >= 9, tail
