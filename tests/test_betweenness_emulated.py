"""The betweenness GPU checks (test_betweenness_gpu.py), reduced in size, on the CPU SIMT emulator (tests/emu): the
unmodified kernels of graph_betweenness.cu bit for bit against the canonical-order oracle without a GPU.  The emulator
library of the other emulated tests does not hold graph_betweenness.cu, so this module compiles it with the emulator's own
pattern rule and links it with that library's objects into a library of its own in a temporary directory."""
import ctypes as C
import glob
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")


@pytest.fixture(scope="module")
def emulated(tmp_path_factory):
    subprocess.check_call(["make", "-C", EMU], stdout=subprocess.DEVNULL)
    subprocess.check_call(["make", "-C", EMU, "graph_betweenness.emu.o"], stdout=subprocess.DEVNULL)
    so = str(tmp_path_factory.mktemp("emu_betweenness") / "libsb200_emu_betweenness.so")
    objs = sorted(glob.glob(os.path.join(EMU, "*.emu.o"))) + [os.path.join(EMU, "emu_runtime.o")]
    subprocess.check_call(["g++", "-shared", "-o", so, *objs, "-pthread", "-ldl"])
    from stract_b200 import _lib
    L = _lib.declare(C.CDLL(so))
    assert b"emulation" in L.sb200_version() and hasattr(L, "sb200_betweenness")
    saved = _lib._LIB
    _lib._LIB = L
    import test_betweenness_gpu as T
    try:
        yield T
    finally:
        _lib._LIB = saved


def test_path_kat_emulated(emulated):
    emulated.check_path_kat()


def test_batch_sizes_emulated(emulated):
    emulated.check_batch_sizes([1, 63, 64, 65, 130], n=160, m=600)


def test_long_rows_emulated(emulated):
    emulated.check_long_rows(fan=1060, extra=400)


def test_diamond_chains_emulated(emulated):
    emulated.check_diamonds()


def test_nofollow_self_loops_and_sinks_emulated(emulated):
    emulated.check_nofollow_self_loops_and_sinks()


def test_refused_inputs_emulated(emulated):
    emulated.check_refused()
