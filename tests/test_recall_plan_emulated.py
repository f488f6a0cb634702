"""The plan recall GPU tests (test_recall_plan_gpu.py), reduced in size, on the CPU SIMT emulator (tests/emu): the unmodified
kernels of bm25_plan.cuh checked against the oracle without a GPU."""
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
    import test_recall_plan_gpu as T
    try:
        yield T
    finally:
        _lib._LIB = saved


def test_plan_docsets_emulated(emulated):
    emulated.check_docsets(max_doc=3_000, nq=30)


def test_plan_recall_emulated(emulated):
    emulated.check_plan_batch(max_doc=2_000, nq=6, k=50)


def test_plan_error_paths_emulated(emulated):
    emulated.check_error_paths(max_doc=500)


def test_plan_phrase_leaves_emulated(emulated):
    emulated.check_phrase_plans(n_docs=400, nq=30)


def test_plan_phrase_exists_not_count_emulated(emulated):
    emulated.check_exists_not_count()


def test_plan_recall_other_stream_emulated(emulated):
    emulated.check_plan_batch(max_doc=2_000, nq=6, k=50, optic=False, order=["UrlForSiteOperator"] + emulated.TO.FIELDS)
