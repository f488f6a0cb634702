"""The size of the pulls' persisting L2 window over the hub rows (the handle option "l2_window_mb") changes where bytes are
cached, never what is computed: every size gives the oracle's result, bit for bit, under each kernel family, across resets of
one handle.  Needs a GPU; test_hyperball_l2_options_emulated.py runs the same functions on the CPU SIMT emulator."""
import ctypes as C

import numpy as np
import pytest

from oracle import hyperball_faithful
from stract_b200 import synth
from stract_b200.webgraph import DeviceGraph, Webgraph

pytestmark = pytest.mark.gpu


def _args(d):
    return (d["from_lo"], d["from_hi"], d["to_lo"], d["to_hi"], d["rel_flags"])


def _check(d, force_mode, window_mbs):
    ref = hyperball_faithful(*_args(d))
    dg = DeviceGraph(Webgraph.from_arrays(*_args(d)))
    try:
        dg.set_policy(force_mode=force_mode)
        for mb in window_mbs:   # one computation per size on the same handle
            dg.set_option("l2_window_mb", mb)
            dg.reset()
            iters, _ = dg.run()
            lo, hi, c = dg.result()
            assert iters == ref["iters"], mb
            assert np.array_equal(lo, ref["ids_lo"]) and np.array_equal(hi, ref["ids_hi"]), mb
            assert np.array_equal(c, ref["centrality"]), f"centrality differs from the oracle with a {mb} MB window"
    finally:
        dg.close()


@pytest.mark.parametrize("force_mode", [-1, 0, 1])
def test_window_sizes_keep_results(force_mode):
    # 3000 nodes: long rows split over several work items next to short rows and rows without in-edges; a 64 KB window
    # covers only the first 1024 rows; 0 (no window) between two sizes
    _check(synth.rmat_graph(3000, 40000, seed=14), force_mode, (16, 0.0625, 0, 24))


def test_window_option_range():
    d = synth.rmat_graph(200, 800, seed=15)
    dg = DeviceGraph(Webgraph.from_arrays(*_args(d)))
    try:
        for bad in (-1, 4096):
            with pytest.raises(Exception):
                dg.set_option("l2_window_mb", bad)
        dg.set_option("l2_window_mb", 0)
        dg.set_option("l2_window_mb", 16)
    finally:
        dg.close()


def _persisting_set_aside():
    """the device's persisting-L2 set-aside, from the CUDA runtime the library runs on (libcudart is loaded with it)"""
    rt = C.CDLL("libcudart.so.12")
    v = C.c_size_t(0)
    assert rt.cudaDeviceGetLimit(C.byref(v), 0x06) == 0   # cudaLimitPersistingL2CacheSize
    return v.value


def test_window_zero_releases_set_aside():
    # "l2_window_mb" 0 gives the persisting set-aside back (the pulls then set no window); a size takes it again.  The
    # computations in between run with each setting and agree with the oracle.
    d = synth.rmat_graph(3000, 40000, seed=16)
    ref = hyperball_faithful(*_args(d))
    dg = DeviceGraph(Webgraph.from_arrays(*_args(d)))
    try:
        for mb, held in ((16, True), (0, False), (0.0625, True), (0, False)):
            dg.set_option("l2_window_mb", mb)
            assert (_persisting_set_aside() > 0) == held, mb
            dg.reset()
            iters, _ = dg.run()
            assert iters == ref["iters"]
            assert np.array_equal(dg.result()[2], ref["centrality"]), mb
            assert (_persisting_set_aside() > 0) == held, mb
    finally:
        dg.close()
