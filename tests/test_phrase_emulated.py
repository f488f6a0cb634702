"""The phrase-query GPU tests (test_phrase_gpu.py), reduced in size, on the CPU SIMT emulator (tests/emu): the unmodified
kernels of bm25_phrase.cuh checked bit-exactly against the oracle without a GPU (see test_bm25_emulated.py)."""
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
    import test_phrase_gpu as T
    try:
        yield T
    finally:
        _lib._LIB = saved


def test_reference_phrase_tests_emulated(emulated):
    emulated.check_reference_phrase_tests()


def test_positions_read_and_errors_emulated(emulated):
    emulated.check_positions_read_kats()
    emulated.check_error_paths()
    emulated.check_term_info_store_positions()


def test_random_phrases_emulated(emulated):
    emulated.check_random_batches(n_docs=700, nq=6, widths=(2, 3, 8))


def test_searcher_and_unchanged_and_or_emulated(emulated):
    emulated.check_searcher_three_segments()
    emulated.check_and_or_unchanged_by_positions()
