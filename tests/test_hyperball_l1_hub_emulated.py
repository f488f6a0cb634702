"""tests/test_hyperball_l1_hub_gpu.py on the CPU SIMT emulator (tests/emu), in-process: every L1 hub budget gives the
oracle's registers and KahanSums after every iteration.  The emulator has no cache, so this checks the option's plumbing
and the split loads' addresses, not their effect."""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")


def test_l1_hub_budgets_against_oracle():
    subprocess.check_call(["make", "-C", EMU], stdout=subprocess.DEVNULL)
    from stract_b200 import _lib
    L = _lib.declare(C.CDLL(os.path.join(EMU, "libsb200_emu.so")))
    saved = _lib._LIB
    _lib._LIB = L
    try:
        import test_hyperball_l1_hub_gpu as T
        for force_mode in (0, 1, 2):
            T.test_l1_hub_budgets_match_oracle_every_iteration(force_mode)
        T.test_l1_hub_option_range()
    finally:
        _lib._LIB = saved
