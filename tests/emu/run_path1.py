"""Runs the path-1 GPU parity functions of tests/test_hyperball_gpu.py against the CPU SIMT emulation of the library
(tests/emu/libsb200_emu.so).  Started as a subprocess by tests/test_hyperball_emulated.py so that a switch read once
per process (SB200_ARENA) can be varied.  argv[1]: "full" or "quick"."""
import ctypes as C
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

from stract_b200 import _lib  # noqa: E402

L = _lib.declare(C.CDLL(os.path.join(HERE, "libsb200_emu.so")))
assert b"emulation" in L.sb200_version()
_lib._LIB = L

import test_hyperball_gpu as T  # noqa: E402

full = (sys.argv[1:] or ["full"])[0] == "full"
T.test_reference_kat_graph()
T.test_rel_flags_and_first_wins()
T.test_edge_cases()
cases = [(60, 300, 1), (2000, 6000, 2), (5000, 60000, 3)] if full else [(2000, 6000, 2)]
for n, e, seed in cases:
    for mode in ((-1, 0, 1, 2) if full else (-1, 2)):
        T.test_random_graph_stepwise(n, e, seed, mode)
if full:
    import test_golden
    test_golden.check_path1_against_golden()   # committed fixtures, no oracle call
    T.test_long_rows_and_hubs()
    import test_round1_late_gpu as late
    late.test_rank_assignment_matches_store_harmonic_order()
if os.environ.get("SB200_ARENA", "1") != "0":   # the slab arena is the default; "0" = stream-ordered pool
    r, u, p, s = (C.c_uint64(0) for _ in range(4))
    L.sb200_arena_stats.argtypes = [C.c_int] + [C.POINTER(C.c_uint64)] * 4
    L.sb200_arena_stats(0, C.byref(r), C.byref(u), C.byref(p), C.byref(s))
    assert s.value > 0 and p.value > 0 and u.value == 0, (r.value, u.value, p.value, s.value)   # used, and everything returned
    print("arena: reserved %d peak %d slabs %d" % (r.value, p.value, s.value))
print("path-1 emulated parity ok")
