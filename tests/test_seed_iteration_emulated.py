"""tests/test_seed_iteration_gpu.py on the CPU SIMT emulator (tests/emu; see tests/test_bm25_emulated.py for what the
emulator is and is not): iteration 0 from the seeds, bit-exact against the oracle, in-process."""
import ctypes as C
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")


@pytest.fixture
def emulated():
    subprocess.check_call(["make", "-C", EMU], stdout=subprocess.DEVNULL)
    from stract_b200 import _lib
    L = _lib.declare(C.CDLL(os.path.join(EMU, "libsb200_emu.so")))
    assert b"emulation" in L.sb200_version()
    saved = _lib._LIB
    _lib._LIB = L
    try:
        import test_seed_iteration_gpu as T
        yield T
    finally:
        _lib._LIB = saved


def test_iteration0_every_register_index(emulated):
    for mode in (-1, 1, 2):
        emulated.test_iteration0_every_register_index(mode)


def test_profile_seed_families_only_in_iteration0(emulated):
    emulated.test_profile_seed_families_only_in_iteration0()


def test_reused_handle_and_bound_state(emulated):
    emulated.test_reused_handle_with_forward_csr()
    emulated.test_bound_state()


def test_group_replicas_after_iteration0(emulated):
    for world in (2, 4):
        emulated.test_group_replicas_after_iteration0(world)
