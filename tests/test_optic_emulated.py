"""The optic docset GPU tests (test_optic_gpu.py), reduced in size, on the CPU SIMT emulator (tests/emu): the unmodified
kernels of bm25_pattern.cuh and k_sig_multi<TMAX, true> checked against the oracle without a GPU."""
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
    import test_optic_gpu as T
    try:
        yield T
    finally:
        _lib._LIB = saved


def test_pattern_docsets_emulated(emulated):
    emulated.check_random_patterns(n_docs=301, n_pat=40)


def test_pattern_error_paths_emulated(emulated):
    emulated.check_error_paths()


def test_optic_recall_batch_emulated(emulated):
    emulated.check_optic_batch(max_doc=2_000, nq=6, k=50)
