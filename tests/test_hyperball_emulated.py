"""Path-1 (HyperBall) kernels and staging on the CPU SIMT emulator (tests/emu; see tests/test_bm25_emulated.py for what
the emulator is and is not).  The parity functions are those of tests/test_hyperball_gpu.py: registers bit-exact after
every iteration, KahanSum bit-exact, output ids and values bit-exact against the oracle, all three kernel families
forced, rows that span several work items.  Besides checking the kernels under the largest lane skew a GPU may show,
this runs both settings of the allocator switch (slab arena vs the driver's stream-ordered pool)."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")


def _run(mode, **env):
    subprocess.check_call(["make", "-C", EMU], stdout=subprocess.DEVNULL)
    e = dict(os.environ)
    for k in ("SB200_ARENA", "SB200_ARENA_SLAB_MB"):
        e.pop(k, None)
    e.update(env)
    r = subprocess.run([sys.executable, os.path.join(EMU, "run_path1.py"), mode], env=e, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "path-1 emulated parity ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
    return r.stdout


def test_default_path_all_kernel_families():
    _run("full")


def test_stream_ordered_pool_instead_of_arena():
    _run("quick", SB200_ARENA="0")


def test_slab_arena():
    out = _run("quick", SB200_ARENA="1", SB200_ARENA_SLAB_MB="4")
    assert "arena: reserved" in out


def test_fused_exchange_by_address_two_and_three_ranks():
    """sb200_hyperball_bind_state + sb200_hyperball_set_publish_targets with several ranks in one emulated process."""
    subprocess.check_call(["make", "-C", EMU], stdout=subprocess.DEVNULL)
    r = subprocess.run([sys.executable, os.path.join(EMU, "run_sharded.py")], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "sharded emulated parity ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])


def test_graph_searches_against_oracle():
    """bit-parallel BFS distances and ApproxHarmonic (graph_bfs.cu) against the oracle, in-process on the emulator"""
    import ctypes as C
    subprocess.check_call(["make", "-C", EMU], stdout=subprocess.DEVNULL)
    from stract_b200 import _lib
    L = _lib.declare(C.CDLL(os.path.join(EMU, "libsb200_emu.so")))
    saved = _lib._LIB
    _lib._LIB = L
    try:
        import test_graph_search_gpu as T
        T.test_distances_match_dijkstra_multi()
        T.test_approx_harmonic_fixed_sample()
        T.test_inbound_similarity_matches_scorer()
        T.test_inbound_similarity_reference_scenarios()
        T.test_distances_reference_scenarios()
    finally:
        _lib._LIB = saved
