"""Betweenness centrality on the device (graph_betweenness.cu) bit for bit against the canonical-order restatement
(betweenness_oracle.py): the reference's path test, batch boundaries, long rows, i32 sigma wrap, NOFOLLOW links,
self-loops, sources that reach nothing, refused inputs, and an R-MAT graph.  test_betweenness_emulated.py runs the same
checks, reduced, on the CPU SIMT emulator."""
import ctypes as C

import numpy as np
import pytest

import betweenness_oracle as B
from stract_b200 import _lib
from stract_b200._lib import Sb200Error
from stract_b200.webgraph import Betweenness, DeviceGraph, Edge, RelFlags, Webgraph

NOFOLLOW = RelFlags.NOFOLLOW


def _device(n, fr, tr, rel=None, seed=0):
    a, ids = B.edge_arrays(n, fr, tr, rel, seed)
    return DeviceGraph(Webgraph.from_arrays(*a), skipped_rel=0), ids


def check(n, fr, tr, src, rel=None, seed=0):
    """Device result for the source ranks `src` (in that order) equals the oracle's: key set, every f64 bit, max_dist."""
    dg, ids = _device(n, fr, tr, rel, seed)
    try:
        lo, hi, c, md = dg.betweenness([ids[s] for s in src])
    finally:
        dg.close()
    cent, reached, omd = B.canonical(n, fr, tr, src)
    keys = np.flatnonzero(reached)
    want_ids = [ids[k] for k in keys]
    got_ids = [(int(h) << 64) | int(l) for l, h in zip(lo, hi)]
    assert got_ids == want_ids
    assert B.same_bits(c, cent[keys]), np.flatnonzero(c.view(np.uint64) != cent[keys].view(np.uint64))[:10]
    assert md == omd
    return dict(zip(keys.tolist(), c.tolist())), md


def check_path_kat():
    g = Webgraph()
    for i in range(4):
        g.insert(Edge.new_test(i, i + 1))
    r = Betweenness.calculate(g)
    assert r.centrality == {0: 0.0, 1: 0.15, 2: 0.2, 3: 0.15, 4: 0.0} and r.max_dist == 4
    check(*B.path(5), [4, 2, 0, 3, 1])


def check_batch_sizes(counts, n=300, m=1500):
    n, fr, tr = B.random_graph(n, m, 21)
    order = np.random.default_rng(5).permutation(np.unique(np.concatenate([fr, tr])))
    for k in counts:
        check(n, fr, tr, order[:k])


def check_long_rows(fan=1100, extra=3000):
    """A hub with `fan` in-links and `fan` out-links (both above CHUNK_EDGES = 1024: several work items per row) in a
    random graph, so the hub's sigma sums several partials and its out-row is walked in several 32-edge steps."""
    n = 2 * fan + 200
    rng = np.random.default_rng(8)
    hub = 0
    ins = np.arange(1, fan + 1, dtype=np.uint32); outs = np.arange(fan + 1, 2 * fan + 1, dtype=np.uint32)
    rf = rng.integers(0, n, extra).astype(np.uint32); rt = rng.integers(0, n, extra).astype(np.uint32)
    fr = np.concatenate([ins, np.full(fan, hub, np.uint32), rf]); tr = np.concatenate([np.full(fan, hub, np.uint32), outs, rt])
    nodes = np.unique(np.concatenate([fr, tr]))
    srcs = np.concatenate([[hub], rng.choice(nodes[1:], 69, replace=False)]).astype(np.uint32)
    check(n, fr, tr, srcs)


def check_diamonds():
    for k in (31, 32):
        n, fr, tr = B.diamonds(k)
        got, md = check(n, fr, tr, [0, 3 * k])
        assert md == 2 * k and got[3 * k - 2] == (-0.25 if k == 31 else -np.inf)
        check(n, fr, tr, [0, 3, 1, 4, 2, 3 * k - 1])


def check_nofollow_self_loops_and_sinks():
    n, fr, tr = B.random_graph(120, 600, 13)                      # self-loops included: no-ops
    assert np.any(fr == tr)
    n = 126                                                         # 120..125: sinks
    fr = np.concatenate([fr, np.arange(0, 60, 10, dtype=np.uint32)]); tr = np.concatenate([tr, np.arange(120, 126, dtype=np.uint32)])
    rel = np.full(fr.size, NOFOLLOW | RelFlags.UGC, np.uint64)    # links the harmonic centrality skips still count here
    check(n, fr, tr, np.arange(0, 120, 2), rel=rel)
    outdeg = np.bincount(fr[fr != tr], minlength=n)
    nodes = np.unique(np.concatenate([fr, tr]))
    sinks = [v for v in nodes if outdeg[v] == 0]
    got, md = check(n, fr, tr, sinks[:3] + [int(nodes[0])] + sinks[3:6])
    # the reference's map for sinks only: each source at 0.0 (one source: 0/0)
    a, _ = B.edge_arrays(n, fr, tr)
    r = Betweenness.calculate(Webgraph.from_arrays(*a), sources=[B.to_ids(n)[2][s] for s in sinks[:2]])
    assert r.max_dist == 0 and sorted(r.centrality.values()) == [0.0, 0.0]


def check_refused():
    n, fr, tr = B.path(6)
    dg, ids = _device(n, fr, tr)
    try:
        with pytest.raises(Sb200Error) as e:
            dg.betweenness([ids[0], 12345])
        assert e.value.code == -1
        with pytest.raises(Sb200Error) as e:
            dg.betweenness([ids[1], ids[2], ids[1]])
        assert e.value.code == -1
        L = _lib.lib()
        lo = np.array([ids[0] & (2**64 - 1)], np.uint64); hi = np.array([ids[0] >> 64], np.uint64)
        out = np.zeros(n, np.uint64); oc = np.zeros(n, np.float64); ln = C.c_uint64(); md = C.c_uint32()
        assert L.sb200_betweenness(dg._h, lo.ctypes.data, hi.ctypes.data, 1, out.ctypes.data, out.ctypes.data, oc.ctypes.data, n - 1,
                                   C.byref(ln), C.byref(md)) == -1
        assert L.sb200_betweenness(dg._h, lo.ctypes.data, hi.ctypes.data, 1, out.ctypes.data, out.ctypes.data, oc.ctypes.data, n,
                                   C.byref(ln), C.byref(md)) == 0 and ln.value == n and md.value == n - 1
        none = dg.betweenness([])
        assert len(none[0]) == 0 and none[3] == 0
    finally:
        dg.close()
    # distances are u8: 254 is the deepest a search may go
    n, fr, tr = B.path(255)
    got, md = check(n, fr, tr, [0])
    assert md == 254
    n, fr, tr = B.path(256)
    dg, ids = _device(n, fr, tr)
    try:
        with pytest.raises(Sb200Error) as e:
            dg.betweenness([ids[1], ids[0]])
        assert e.value.code == -4
        assert dg.betweenness([ids[1]])[3] == 254     # the handle stays usable
    finally:
        dg.close()


def _arena_in_use():
    L = _lib.lib()
    L.sb200_arena_stats.restype = C.c_int
    L.sb200_arena_stats.argtypes = [C.c_int] + [C.POINTER(C.c_uint64)] * 4
    v = [C.c_uint64() for _ in range(4)]
    assert L.sb200_arena_stats(0, *[C.byref(x) for x in v]) == 0
    return v[1].value


@pytest.mark.gpu
def test_path_kat():
    check_path_kat()


@pytest.mark.gpu
def test_batch_sizes():
    check_batch_sizes([1, 63, 64, 65, 130, 300])


@pytest.mark.gpu
def test_long_rows():
    check_long_rows()


@pytest.mark.gpu
def test_diamond_chains_wrap_i32():
    check_diamonds()


@pytest.mark.gpu
def test_nofollow_self_loops_and_sinks():
    check_nofollow_self_loops_and_sinks()


@pytest.mark.gpu
def test_refused_inputs():
    check_refused()


@pytest.mark.gpu
def test_rmat_bit_exact_and_arena_returns():
    from stract_b200 import synth
    d = synth.rmat_graph(100_000, 1_000_000, seed=7)
    a = (d["from_lo"], d["from_hi"], d["to_lo"], d["to_hi"], d["rel_flags"])
    ids_lo, ids_hi, fr, tr = B.rank_links(*a[:4])
    n = len(ids_lo)
    src = np.random.default_rng(3).permutation(n)[:300].astype(np.uint32)
    dg = DeviceGraph(Webgraph.from_arrays(*a), skipped_rel=0)
    try:
        before = _arena_in_use()
        lo, hi, c, md = dg.betweenness([(int(ids_hi[s]) << 64) | int(ids_lo[s]) for s in src])
        assert _arena_in_use() == before
    finally:
        dg.close()
    cent, reached, omd = B.canonical(n, fr, tr, src)
    keys = np.flatnonzero(reached)
    assert np.array_equal(lo, ids_lo[keys]) and np.array_equal(hi, ids_hi[keys])
    assert B.same_bits(c, cent[keys]) and md == omd
    assert len(keys) > n // 2 and np.count_nonzero(c) > 1000
