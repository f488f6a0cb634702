"""The LambdaMART GPU tests (test_lambdamart_gpu.py), reduced in size, on the CPU SIMT emulator (tests/emu): the unmodified
k_lambdamart of lambdamart.cu checked against tests/lambdamart_oracle.py without a GPU.  The emulator library of the other
emulated tests does not hold lambdamart.cu, so this module compiles it with the emulator's own pattern rule and links it with
that library's objects into a library of its own in a temporary directory."""
import ctypes as C
import glob
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")


@pytest.fixture(scope="module")
def emulated(tmp_path_factory):
    subprocess.check_call(["make", "-C", EMU], stdout=subprocess.DEVNULL)
    # -B: the pattern rule does not list the LambdaMART header among its prerequisites
    subprocess.check_call(["make", "-C", EMU, "-B", "lambdamart.emu.o"], stdout=subprocess.DEVNULL)
    so = str(tmp_path_factory.mktemp("emu_lambdamart") / "libsb200_emu_lambdamart.so")
    objs = sorted(glob.glob(os.path.join(EMU, "*.emu.o"))) + [os.path.join(EMU, "emu_runtime.o")]
    subprocess.check_call(["g++", "-shared", "-o", so, *objs, "-pthread", "-ldl"])
    from stract_b200 import _lib
    L = _lib.declare(C.CDLL(so))
    assert b"emulation" in L.sb200_version() and hasattr(L, "sb200_lambdamart_predict")
    saved = _lib._LIB
    _lib._LIB = L
    import test_lambdamart_gpu as T
    try:
        yield T
    finally:
        _lib._LIB = saved


def test_lambdamart_fixture_emulated(emulated):
    emulated.check_fixture(n_rows=300)


def test_lambdamart_synthetic_emulated(emulated):
    emulated.check_synthetic([(1, 1, 2, 0, 40), (3, 60, (2, 63), 7, 150), (5, 12, 255, 0, 130)])


def test_lambdamart_chain_and_global_tree_emulated(emulated):
    emulated.check_chain(300, 40)
    # 3 000 leaves: 72 KB, above the 32 KB shared tree buffer
    rng = np.random.default_rng(12)
    import lambdamart_oracle as O
    text, th = O.random_model(rng, 2, 3_000)
    emulated.check_model(text, O.random_rows(rng, 140, th))


def test_lambdamart_batch_sizes_emulated(emulated):
    emulated.check_batch_sizes([1, 31, 32, 33, 127, 128, 129])


def test_lambdamart_load_errors_emulated(emulated):
    emulated.check_load_errors()


def test_lambdamart_bad_args_emulated(emulated):
    emulated.check_bad_args()


def test_lambdamart_recall_stage_emulated(emulated):
    emulated.check_pipeline(n_docs=400, nq=4, k=30, long_doc=100)
