"""The recall-webpage GPU tests (test_recall_webpages_gpu.py), reduced in size, on the CPU SIMT emulator (tests/emu): the
unmodified kernels of bm25_webpage.cuh checked against tests/webpage_oracle.py without a GPU."""
import ctypes as C
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")


@pytest.fixture(scope="module")
def emulated():
    subprocess.check_call(["make", "-C", EMU], stdout=subprocess.DEVNULL)
    from stract_b200 import _lib
    L = _lib.declare(C.CDLL(os.path.join(EMU, "libsb200_emu.so")))
    assert b"emulation" in L.sb200_version()
    saved = _lib._LIB
    _lib._LIB = L
    import test_recall_webpages_gpu as T
    try:
        yield T
    finally:
        _lib._LIB = saved


def test_webpages_emulated(emulated):
    # doc 0 of CleanBody alternates two terms 850 times each: 1 700 positions, above the shared-memory buffer
    emulated.check_webpages(n_docs=500, nq=16, k=12, long_doc=1_700)


def test_webpages_optic_emulated(emulated):
    emulated.check_webpages(n_docs=500, nq=12, k=12, long_doc=300, optic=True, seed=8)


def test_webpages_recall_stage_emulated(emulated):
    emulated.check_recall_stage(n_docs=400, nq=8, k=10, long_doc=200)


def test_webpages_error_paths_emulated(emulated):
    emulated.check_error_paths(n_docs=300)


def test_webpages_hand_positions_emulated(emulated):
    emulated.check_hand_positions()
