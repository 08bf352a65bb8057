"""tests/test_mask_planes_gpu.py on the CPU emulator: the library compiled for tests/emu (same kernel and
host sources) behind the real C-ABI, in a child process, as tests/test_c_abi_on_emulator.py does for the
rest of the GPU parity suite."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_sweep  # noqa: E402


def test_mask_planes_suite_on_the_emulated_library():
    got = emu_sweep.run_suite("tests/test_mask_planes_gpu.py")
    assert got["passed"] >= 5, got
