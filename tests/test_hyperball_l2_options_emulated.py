"""tests/test_hyperball_l2_options_gpu.py on the CPU SIMT emulator (tests/emu), in-process: every size of the pulls' L2
window gives the oracle's result.  The emulator has no cache, so this checks the option's plumbing, not its effect."""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")


def test_window_sizes_against_oracle():
    subprocess.check_call(["make", "-C", EMU], stdout=subprocess.DEVNULL)
    from stract_b200 import _lib
    L = _lib.declare(C.CDLL(os.path.join(EMU, "libsb200_emu.so")))
    saved = _lib._LIB
    _lib._LIB = L
    try:
        import test_hyperball_l2_options_gpu as T
        for force_mode in (-1, 0, 1):
            T.test_window_sizes_keep_results(force_mode)
        T.test_window_option_range()
    finally:
        _lib._LIB = saved
