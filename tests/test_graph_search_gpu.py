"""The other graph kernels over the resident CSR (SURVEY 8(f) rank 4): shortest-path distances (dijkstra_multi with unit
costs, incl. its max_dist cut-off and reversed searches) exact against the oracle; ApproxHarmonic for a fixed sample against
the oracle's f64 sums (identical f32 terms) and within f32 accumulation error of the reference-shaped f32 sums."""
import numpy as np
import pytest

import oracle
from stract_b200 import synth
from stract_b200.webgraph import DeviceGraph, Webgraph

pytestmark = pytest.mark.gpu


def _graph(seed=3, nodes=4000, edges=30000):
    d = synth.rmat_graph(nodes, edges, seed=seed)
    a = (d["from_lo"], d["from_hi"], d["to_lo"], d["to_hi"], d["rel_flags"])
    ids_lo, ids_hi, fr, tr = oracle.graph_links(*a, skip_mask=0)
    keep = fr != tr          # a self-loop never shortens a path; the device CSR drops it
    return a, ids_lo, ids_hi, fr[keep], tr[keep]


def test_distances_match_dijkstra_multi():
    a, ids_lo, ids_hi, fr, tr = _graph()
    n = len(ids_lo)
    dg = DeviceGraph(Webgraph.from_arrays(*a), skipped_rel=0)      # every link, as ForwardlinksQuery sees them
    try:
        assert dg.info()["n_nodes"] == n
        rng = np.random.default_rng(1)
        src = rng.choice(n, 70, replace=False).astype(np.uint32)
        ids = [(int(ids_hi[s]) << 64) | int(ids_lo[s]) for s in src]
        for reversed_ in (False, True):
            for max_dist in (None, 2, 7):
                for lo in (0, 64):       # 64 searches fill the bit word; the rest goes in a second call
                    part = slice(lo, min(lo + 64, len(src)))
                    want = oracle.graph_distances(n, fr, tr, src[part], None, max_dist, reversed_)
                    got = dg.distances(ids[part], None, 0 if max_dist is None else max_dist, reversed_)
                    assert np.array_equal(got, want), (reversed_, max_dist, lo)
        # several sources per search (dijkstra_multi's `sources` slice) + an id that is not a node
        groups = np.array([0, 0, 0, 1, 1, 2], np.uint32)
        want = oracle.graph_distances(n, fr, tr, src[:6], groups, 3, False)
        got = dg.distances(ids[:6] + [12345], np.concatenate([groups, [2]]).astype(np.uint32), 3, False)
        assert np.array_equal(got, want)
        assert (want[0] <= 4).sum() > 3 and want.max() == 255     # the cut-off reports distances up to max_dist + 1
    finally:
        dg.close()


def test_approx_harmonic_fixed_sample():
    a, ids_lo, ids_hi, fr, tr = _graph(seed=9, nodes=6000, edges=60000)
    n = len(ids_lo)
    dg = DeviceGraph(Webgraph.from_arrays(*a), skipped_rel=0)
    try:
        rng = np.random.default_rng(2)
        outdeg = np.bincount(fr, minlength=n)
        cand = np.flatnonzero(outdeg > 0)                       # random_page_nodes_with_outgoing
        k = int(np.ceil(np.log2(n) / 0.3 ** 2))                 # approx_harmonic.rs:50
        src = rng.choice(cand, k, replace=False).astype(np.uint32)
        ids = [(int(ids_hi[s]) << 64) | int(ids_lo[s]) for s in src]
        w32, w64 = oracle.approx_harmonic(n, fr, tr, src, 7, n)
        lo, hi, c = dg.approx_harmonic(ids, 7, n)
        reached = np.flatnonzero(w64 != 0.0)
        assert np.array_equal(lo, ids_lo[reached]) and np.array_equal(hi, ids_hi[reached])
        # Bit-exact although the two sum in different orders: every term is the f32 value norm / d, d <= 8, so each is an
        # integer multiple of the smallest term's ulp, and a sum of k samples of them stays far below 2^53 such ulps --
        # the device's per-level popcount * term additions and the oracle's per-source additions are both exact in f64.
        assert np.array_equal(c.view(np.uint64), w64[reached].view(np.uint64))
        assert np.allclose(c, w32[reached].astype(np.float64), rtol=2e-5)    # the reference-shaped f32 accumulation
    finally:
        dg.close()


def test_inbound_similarity_matches_scorer():
    """inbound_similarity::Scorer over the resident CSR: bit-exact f64 scores, incl. the bloom pre-filter's false negatives,
    self-links as in-neighbours, self_score, ids that are not nodes, empty lists and more than 64 liked nodes (two passes)."""
    d = synth.rmat_graph(3000, 40000, seed=21)
    a = [d["from_lo"].copy(), d["from_hi"].copy(), d["to_lo"].copy(), d["to_hi"].copy(), d["rel_flags"].copy()]
    for k in range(0, 400, 7):                      # plant self-links
        a[2][k] = a[0][k]; a[3][k] = a[1][k]
    a = tuple(a)
    ids_lo, ids_hi, fr, tr = oracle.graph_links(*a, skip_mask=0)
    n = len(ids_lo)
    assert (fr == tr).sum() > 20
    dg = DeviceGraph(Webgraph.from_arrays(*a), skipped_rel=0)
    try:
        rng = np.random.default_rng(5)
        indeg = np.bincount(tr, minlength=n)
        popular = np.argsort(-indeg)[:300]
        selfers = np.unique(fr[fr == tr])
        def ids_of(ranks):
            return [((int(ids_hi[r]) << 64) | int(ids_lo[r])) if r != 0xFFFFFFFF else (1 << 100) + 12345 for r in ranks]
        cases = []
        liked = np.concatenate([rng.choice(popular, 20, replace=False), selfers[:5]]).astype(np.uint32)
        disliked = np.concatenate([rng.choice(popular, 9, replace=False), selfers[5:8], [0xFFFFFFFF]]).astype(np.uint32)
        cand = np.concatenate([rng.choice(n, 500, replace=False), liked[:4], disliked[:3], selfers[:10], [0xFFFFFFFF]]).astype(np.uint32)
        cases.append((liked, disliked, cand, False, 1.0))
        cases.append((liked, disliked, cand, True, 0.25))
        cases.append((rng.choice(popular, 150, replace=False).astype(np.uint32), rng.choice(n, 70, replace=False).astype(np.uint32), cand, True, 1.0))
        cases.append((np.zeros(0, np.uint32), disliked, cand, True, 1.0))
        cases.append((liked, np.zeros(0, np.uint32), cand[:1], False, 1.0))
        cases.append((np.zeros(0, np.uint32), np.zeros(0, np.uint32), cand[:40], False, 1.0))
        nonzero = 0
        for li, di, ca, norm, ss in cases:
            want = oracle.inbound_similarity(ids_lo, ids_hi, fr, tr, li, di, ca, norm, ss)
            got = dg.inbound_similarity(ids_of(li), ids_of(di), ids_of(ca), norm, ss)
            assert got.tobytes() == want.tobytes(), (len(li), len(di), norm, np.flatnonzero(got != want)[:5])
            nonzero += int((want != float(len(di))).sum())
        assert nonzero > 200
    finally:
        dg.close()


def _ids(n, seed=77):
    rng = np.random.default_rng(seed)
    lo = rng.integers(1, 2 ** 63, n, dtype=np.uint64); hi = rng.integers(1, 2 ** 63, n, dtype=np.uint64)
    return [(int(h) << 64) | int(l) for l, h in zip(lo, hi)]


def _graph_from(edges, rel=None):
    fl = np.array([f & ((1 << 64) - 1) for f, _ in edges], np.uint64); fh = np.array([f >> 64 for f, _ in edges], np.uint64)
    tl = np.array([t & ((1 << 64) - 1) for _, t in edges], np.uint64); th = np.array([t >> 64 for _, t in edges], np.uint64)
    r = np.zeros(len(edges), np.uint64) if rel is None else np.array(rel, np.uint64)
    return fl, fh, tl, th, r


def _scores_both(arrays, skip, liked, disliked, cands, normalized=False):
    """(device scores, oracle scores) for the same handle-shaped input"""
    ids_lo, ids_hi, fr, tr = oracle.graph_links(*arrays, skip_mask=skip)
    pos = {(int(h) << 64) | int(l): i for i, (l, h) in enumerate(zip(ids_lo, ids_hi))}
    rk = lambda xs: np.array([pos.get(x, 0xFFFFFFFF) for x in xs], np.uint32)
    want = oracle.inbound_similarity(ids_lo, ids_hi, fr, tr, rk(liked), rk(disliked), rk(cands), normalized)
    dg = DeviceGraph(Webgraph.from_arrays(*arrays), skipped_rel=skip)
    try:
        got = dg.inbound_similarity(liked, disliked, cands, normalized)
    finally:
        dg.close()
    assert got.tobytes() == want.tobytes()
    return got


def test_inbound_similarity_reference_scenarios():
    """The reference's own tests for this path, on the oracle AND the device: `it_favors_liked_hosts`
    (ranking/inbound_similarity.rs:168-236), the BitVec cases `simple` / `zero_sim` / `empty_sim` / `low_sim`
    (ranking/bitvec_similarity.rs:222-295, sets given as in-neighbour sets of two nodes) and `test_ignores_no_follow` (:297-330)."""
    from stract_b200.webgraph import RelFlags
    a, b, c, d, e, z = _ids(6)
    edges = [(a, b), (c, d), (a, e), (z, a), (z, b), (z, c), (z, d), (z, d), (z, e)]
    s = _scores_both(_graph_from(edges), 0, [b], [], [e, d])
    assert s[0] > s[1]                                             # it_favors_liked_hosts
    # BitVec cases: node X has in-neighbours = the set a, node Y the set b
    def bitvec_sim(set_a, set_b, n_nodes):
        ids = _ids(n_nodes + 2, seed=5)
        x, y, src = ids[0], ids[1], ids[2:]
        ed = [(src[i], x) for i in set_a] + [(src[i], y) for i in set_b]
        ed += [(x, src[0]), (y, src[0])]                             # X and Y are nodes of the graph even with an empty in-neighbour set
        return _scores_both(_graph_from(ed), 0, [x], [], [y])[0]
    naive = lambda sa, sb: len(set(sa) & set(sb)) / (np.sqrt(len(sa)) * np.sqrt(len(sb)))
    sa, sb = list(range(1000, 1010)), list(range(1000, 1008))
    assert abs(bitvec_sim(sa, sb, 1010) - naive(sa, sb)) < 0.1     # simple
    assert bitvec_sim([], list(range(300)), 300) == 0.0            # zero_sim (one side empty)
    assert bitvec_sim([], [], 4) == 0.0                            # empty_sim
    sa, sb = list(range(3000, 3010)), list(range(0, 3008))
    assert naive(sa, sb) < 0.05 and abs(bitvec_sim(sa, sb, 3010) - naive(sa, sb)) < 0.1   # low_sim (3 000 instead of 100 000 common in-links)
    # test_ignores_no_follow: A -nofollow-> B, A -> C: with NOFOLLOW in the handle's skip mask sim(B, C) is 0
    A, B, C = _ids(3, seed=9)
    arr = _graph_from([(A, B), (A, C)], rel=[RelFlags.NOFOLLOW, 0])
    assert _scores_both(arr, RelFlags.NOFOLLOW, [B], [], [C])[0] == 0.0
    assert _scores_both(arr, 0, [B], [], [C])[0] == 1.0            # and counted when it is not skipped: both have exactly {A}


def test_distances_reference_scenarios():
    """webgraph/tests.rs:57-137: `distance_calculation`, `nonexisting_node`, `reversed_distance_calculation` on the reference's
    five-edge test graph (A->B, B->C, A->C, C->A, D->C), oracle and device."""
    A, B, C, D, E = _ids(5, seed=31)
    arrays = _graph_from([(A, B), (B, C), (A, C), (C, A), (D, C)])
    ids_lo, ids_hi, fr, tr = oracle.graph_links(*arrays, skip_mask=0)
    pos = {(int(h) << 64) | int(l): i for i, (l, h) in enumerate(zip(ids_lo, ids_hi))}
    dg = DeviceGraph(Webgraph.from_arrays(*arrays), skipped_rel=0)
    try:
        def both(src, rev):
            want = oracle.graph_distances(4, fr, tr, np.array([pos[src]], np.uint32), None, None, rev)[0]
            got = dg.distances([src], None, 0, rev)[0]
            assert np.array_equal(got, want)
            return {k: int(got[pos[k]]) for k in (A, B, C, D)}
        d = both(D, False)
        assert (d[C], d[A], d[B]) == (1, 2, 3)                                  # distance_calculation
        d = both(D, True)
        assert (d[C], d[A], d[B]) == (255, 255, 255)                            # reversed from D: nothing links to D
        d = both(A, True)
        assert (d[C], d[D], d[B]) == (1, 2, 2)                                  # reversed_distance_calculation
        for rev in (False, True):                                               # nonexisting_node: no distances at all
            assert (dg.distances([E], None, 0, rev)[0] == 255).all()
    finally:
        dg.close()
