"""HyperBall and the graph searches over the graph's structural range (tests/graph_range.py): rows of exactly 1 .. 16 385
in-edges around the quad / warp / multi-item boundaries, a hub of 69 work items, more multi-item rows than one merge CTA
takes, a 70 000-edge push source, first-wins duplicates, self-links, the all-ones id and ids sharing a half, and a
300-node chain that runs HyperBall past 256 iterations and BFS into the 254-level cap of u8 distances.  Needs a GPU.

Every comparison is exact: HyperLogLog registers and KahanSum (sum, err) after every iteration, distances, ApproxHarmonic's
f64 sums and inbound-similarity scores by bits.  tests/test_graph_range_emulated.py runs the same check_* functions,
reduced, on the CPU emulator."""
import numpy as np
import pytest

import graph_range as G
import oracle
from oracle import DenseHyperBall, hyperball_faithful
from stract_b200._lib import Sb200Error
from stract_b200.webgraph import SKIPPED_REL, DeviceGraph, DeviceGroup, HarmonicCentrality, Webgraph

pytestmark = pytest.mark.gpu
SB200_ERANGE = -4
NON_NODE = (1 << 100) + 12345      # the one id that is not a node (the oracles take it as rank 0xFFFFFFFF)
NO_RANK = 0xFFFFFFFF


def _webgraph(fx):
    return Webgraph.from_arrays(*G.args(fx))


def _id(ids_lo, ids_hi, r):
    return NON_NODE if r == NO_RANK else (int(ids_hi[r]) << 64) | int(ids_lo[r])


def _launches(dg):
    return {p["name"]: p["launches"] for p in dg.profile()}


# ---------------------------------------------------------------------------------------------------------- HyperBall
def _stepwise(dg, orc, max_steps=100_000):
    """step the device handle and the dense oracle together: registers and KahanSum bit-exact after every iteration,
    ids and centralities bit-exact at the end; returns the iteration count"""
    lo, hi = dg.node_ids()
    olo, ohi = orc.ids()
    assert np.array_equal(lo, olo) and np.array_equal(hi, ohi)
    assert np.array_equal(dg.registers(), orc.registers())
    for it in range(max_steps):
        st = dg.step()
        nch = orc.step()
        assert st["n_changed"] == nch, (it, st, nch)
        assert np.array_equal(dg.registers(), orc.registers()), f"registers differ after iteration {it} (mode {st['mode']})"
        s, e = dg.kahan()
        os_, oe = orc.kahan()
        assert np.array_equal(s.view(np.uint64), os_.view(np.uint64)) and np.array_equal(e.view(np.uint64), oe.view(np.uint64)), \
            f"KahanSum differs after iteration {it}"
        if nch == 0:
            break
    glo, ghi, gc = dg.result()
    r = orc.result()
    assert np.array_equal(glo, r["ids_lo"]) and np.array_equal(ghi, r["ids_hi"])
    assert np.array_equal(gc.view(np.uint64), r["centrality"].view(np.uint64))
    return it + 1


def check_hyperball_stepwise(fx, modes=(-1, 0, 1, 2)):
    G.self_check(fx, SKIPPED_REL)
    orc = DenseHyperBall(*G.args(fx), threads=8)
    try:
        assert orc.n_nodes == fx["n"]
        for mode in modes:
            dg = DeviceGraph(_webgraph(fx))
            try:
                dg.set_policy(force_mode=mode)
                dg.set_profiling(True)
                orc.reset()
                iters = _stepwise(dg, orc)
                assert iters > G.CHAIN_LEN
                ran = _launches(dg)
                if mode == 2:
                    assert ran["k_push"] > 0, ran
                else:
                    for k in ("k_pull_merge", "k_pull_warp<seed>", "k_pull_quad<seed>"):
                        assert ran[k] > 0, (mode, ran)
                    assert ran["k_pull_merge"] == ran["k_pull_warp<seed>"] + ran["k_pull_warp<dense>"] + ran["k_pull_warp<frontier>"]
                if mode == -1:
                    # a reused handle: the push branch builds the source-major CSR lazily once the frontier is small
                    dg.reset()
                    dg.set_profiling(True)
                    orc.reset()
                    assert _stepwise(dg, orc) == iters
                    ran = _launches(dg)
                    assert ran["k_push"] > 0 and ran["k_pull_merge"] > 0 and ran["k_pull_warp<seed>"] > 0, ran
            finally:
                dg.close()
    finally:
        orc.close()


def check_sharded_group(fx, worlds=(2, 3), modes=(-1, 2)):
    a = G.args(fx)
    ref = hyperball_faithful(*a)
    dense = DenseHyperBall(*a, threads=8)
    dense.run()
    want = dense.registers()
    dense.close()
    for world in worlds:
        for mode in modes:
            grp = DeviceGroup(_webgraph(fx), [0] * world)
            try:
                for h in grp.ranks:
                    h.set_policy(force_mode=mode)
                own = [h.ownership() for h in grp.ranks]
                assert np.array_equal(np.sum([o for o, _ in own], axis=0), np.ones(fx["n"], np.uint8))
                need = [o.astype(bool) | (((m >> r) & 1) == 1) for r, (o, m) in enumerate(own)]
                # the multi-item rows (internal rows 0..47, in 32-row blocks) belong to more than one rank
                for rep in range(2):
                    if rep:
                        grp.reset()
                    t, _ = grp.run()
                    lo, hi, c = grp.result()
                    assert t == ref["iters"], (world, mode, rep, t, ref["iters"])
                    assert np.array_equal(lo, ref["ids_lo"]) and np.array_equal(hi, ref["ids_hi"])
                    assert np.array_equal(c.view(np.uint64), ref["centrality"].view(np.uint64)), (world, mode, rep)
                    for r, h in enumerate(grp.ranks):
                        assert np.array_equal(h.registers()[need[r]], want[need[r]]), (world, mode, rep, r)
            finally:
                grp.close()


def check_long_run(fx):
    a = G.args(fx)
    ref = hyperball_faithful(*a)
    assert ref["iters"] > 256, ref["iters"]
    got = HarmonicCentrality.calculate(_webgraph(fx))
    assert got.iterations == ref["iters"] and len(got.stats) == 256
    assert np.array_equal(got.ids_lo, ref["ids_lo"]) and np.array_equal(got.ids_hi, ref["ids_hi"])
    assert np.array_equal(got.values.view(np.uint64), ref["centrality"].view(np.uint64))
    dg = DeviceGraph(_webgraph(fx))
    orc = DenseHyperBall(*a)
    try:
        done, stats = dg.run(cap=256)
        assert done == ref["iters"] and len(stats) == 256
        dg.reset()
        assert _stepwise(dg, orc) == ref["iters"]
    finally:
        dg.close()
        orc.close()


def test_hyperball_stepwise_range_graph():
    check_hyperball_stepwise(G.range_graph(1, "full"))


def test_sharded_group_range_graph():
    check_sharded_group(G.range_graph(1, "full"))


def test_long_run_chain():
    check_long_run(G.chain_graph(300))


# ------------------------------------------------------------------------------------------------------------ distances
def _search_links(fx, mask):
    ids_lo, ids_hi, fr, tr = G.links(fx, mask)
    keep = fr != tr          # a self-loop never shortens a path; the device CSR drops it
    return ids_lo, ids_hi, fr[keep], tr[keep]


def range_sources(fx, mask, rng):
    """64 groups of source ranks: one search per multi-item row and per single-item warp row, seeded at the in-neighbour
    that ends a work item (a row keeps its sources in ascending rank order, so positions 1023 and deg - 1 are the last
    edges of an item); groups with duplicated and non-node sources; group 62 only a non-node id; group 63 on the hubs."""
    ids_lo, _, fr, tr = _search_links(fx, mask)
    n = len(ids_lo)
    indeg = np.bincount(tr, minlength=n)
    order = np.argsort(tr, kind="stable")
    ptr = np.concatenate([[0], np.cumsum(indeg)])
    ins = lambda r: np.sort(fr[order[ptr[r]:ptr[r + 1]]])
    rows = np.argsort(-indeg, kind="stable")
    multi = [r for r in rows if indeg[r] > G.CHUNK_EDGES]
    single = [r for r in rows if G.QUAD_MAX_DEG < indeg[r] <= G.CHUNK_EDGES]
    src, grp = [], []
    for g, r in enumerate(multi[:48]):
        src.append(ins(r)[G.CHUNK_EDGES - 1]); grp.append(g)
    for g, r in enumerate(single[:6], start=48):
        src.append(ins(r)[-1]); grp.append(g)
    pool = rng.choice(n, 24, replace=False)
    for k, g in enumerate(range(54, 62)):
        s = list(pool[3 * k:3 * k + 3])
        if k % 2 == 0:
            s.append(s[0])            # duplicated within the group
        if k % 4 == 1:
            s.append(NO_RANK)         # an id that is not a node
        src += s; grp += [g] * len(s)
    src.append(NO_RANK); grp.append(62)
    hub = G.rank_of(fx, mask, G.HUB)
    src += [hub, G.rank_of(fx, mask, 16), hub]; grp += [63, 63, 63]
    return np.array(src, np.uint32), np.array(grp, np.uint32), multi[:48]


def chain_sources(fx, mask):
    core, r = fx["core"], lambda i: G.rank_of(fx, mask, i)
    src = [r(0), r(core), r(core + 5), r(core + 5), NO_RANK, r(core + fx["length"] - 1), r(1)]
    grp = [0, 1, 2, 2, 2, 62, 63]
    return np.array(src, np.uint32), np.array(grp, np.uint32)


def check_distances(fx, src, grp, mask, max_dists=(None, 1, 7, 253)):
    ids_lo, ids_hi, fr, tr = _search_links(fx, mask)
    n = len(ids_lo)
    ids = [_id(ids_lo, ids_hi, s) for s in src]
    assert int(grp.max()) == 63 and len(set(grp.tolist())) == 64 or "core" in fx
    dg = DeviceGraph(_webgraph(fx), skipped_rel=mask)
    out = {}
    try:
        assert dg.info()["n_nodes"] == n
        for rev in (False, True):
            for md in max_dists:
                want = oracle.graph_distances(n, fr, tr, src, grp, md, rev)
                got = dg.distances(ids, grp, 0 if md is None else md, rev)
                assert got.shape == (64, n)
                bad = np.argwhere(got != want)
                assert bad.size == 0, (rev, md, bad[:8].tolist(), [(int(got[g, v]), int(want[g, v])) for g, v in bad[:8]])
                assert (want[63] < 255).sum() > 1
                out[(rev, md)] = want
        with pytest.raises(Sb200Error) as e:
            dg.distances(ids, grp, 254, False)
        assert e.value.code == SB200_ERANGE
    finally:
        dg.close()
    return out


def check_range_distances(fx, mask):
    src, grp, item_rows = range_sources(fx, mask, np.random.default_rng(4))
    want = check_distances(fx, src, grp, mask)
    # the item-end searches reach their row at distance 1 through that one edge
    assert all(want[(False, 1)][g][r] == 1 for g, r in enumerate(item_rows))


def check_chain_distances(fx, mask):
    src, grp = chain_sources(fx, mask)
    want = check_distances(fx, src, grp, mask)
    core, c = fx["core"], lambda k: G.rank_of(fx, mask, fx["core"] + k)
    for md in (None, 253):
        d = want[(False, md)]
        assert d[0][c(252)] == 253 and d[0][c(253)] == 254 and d[0][c(254)] == 255 and d[0][c(fx["length"] - 1)] == 255
    assert want[(True, None)][62][c(fx["length"] - 1 - 254)] == 254
    assert want[(True, None)][62][c(fx["length"] - 1 - 255)] == 255


@pytest.mark.parametrize("mask", [0, SKIPPED_REL])
def test_distances_range_graph(mask):
    check_range_distances(G.range_graph(1, "full"), mask)


def test_distances_chain():
    check_chain_distances(G.chain_graph(300), 0)


# ------------------------------------------------------------------------------------------------------ ApproxHarmonic
def check_approx_harmonic(fx, mask, sizes=(1, 63, 64, 65, 130), max_dists=(1, 7, 253), big_num_nodes=(1, 65), seed=6):
    """Ids equal and centralities bit-exact against the oracle's f64 sums.  Every term is the f32 value norm / d rounded
    to f32, d <= max_dist + 1 <= 254, so every term is an integer multiple of the ulp of the smallest term and at most
    2^24 * 2^9 of those ulps; a sum of <= 130 samples * 64 bits of such terms stays below 2^53 ulps.  Both the device's
    per-level popcount * term additions and the oracle's per-source additions are therefore exact in f64, in any order."""
    ids_lo, ids_hi, fr, tr = _search_links(fx, mask)
    n = len(ids_lo)
    outdeg = np.bincount(fr, minlength=n)
    cand = np.flatnonzero(outdeg > 0)
    rng = np.random.default_rng(seed)
    dg = DeviceGraph(_webgraph(fx), skipped_rel=mask)
    try:
        runs = [(k, md, n) for k in sizes for md in max_dists] + [(k, 7, (1 << 24) + 1) for k in big_num_nodes]
        for k, md, nn in runs:
            src = rng.choice(cand, k, replace=k > cand.size).astype(np.uint32)
            if k >= 63:
                src[[5, 40]] = NO_RANK                                  # ids that are not nodes count in the sample
                src[k - 1] = G.rank_of(fx, mask, G.HUB) if "hub" in fx else src[k - 1]
            ids = [_id(ids_lo, ids_hi, s) for s in src]
            w32, w64 = oracle.approx_harmonic(n, fr, tr, src, md, nn)
            lo, hi, c = dg.approx_harmonic(ids, md, nn)
            reached = np.flatnonzero(w64 != 0.0)
            assert reached.size > 0
            assert np.array_equal(lo, ids_lo[reached]) and np.array_equal(hi, ids_hi[reached]), (k, md, nn)
            bad = np.flatnonzero(c.view(np.uint64) != w64[reached].view(np.uint64))
            assert bad.size == 0, (k, md, nn, [(float(c[i]), float(w64[reached][i])) for i in bad[:5]])
            assert np.allclose(c, w32[reached].astype(np.float64), rtol=2e-5)    # the reference-shaped f32 accumulation
    finally:
        dg.close()


def test_approx_harmonic_range_graph():
    check_approx_harmonic(G.range_graph(1, "full"), 0)


def test_approx_harmonic_chain():
    check_approx_harmonic(G.chain_graph(300), 0, sizes=(1, 64, 65), max_dists=(253,), big_num_nodes=(65,))


# -------------------------------------------------------------------------------------------------- inbound similarity
def _blooms(ids_lo, fr, tr, ranks):
    """VeryJankyBloomFilter (16 x 64 bit over the low 64 bits of the ids) of the in-neighbour set of each rank: [len(ranks), 16]"""
    out = np.zeros((len(ranks), 16), np.uint64)
    for i, r in enumerate(ranks):
        h = ids_lo[np.unique(fr[tr == r])] * np.uint64(11400714819323198549)
        np.bitwise_or.at(out[i], (h % np.uint64(16)).astype(np.int64), np.uint64(1) << (h % np.uint64(64)))
    return out


def _popcount(a):
    return np.unpackbits(np.ascontiguousarray(a).view(np.uint8), axis=-1).sum(axis=-1)


def _prefilter_counts(ids_lo, fr, tr, targets, cands):
    """(rejected, accepted) (target, candidate) pairs of BitVec::sim's bloom pre-filter, both sets non-empty"""
    t = np.unique(targets[targets != NO_RANK]); c = np.unique(cands[cands != NO_RANK])
    bt, bc = _blooms(ids_lo, fr, tr, t), _blooms(ids_lo, fr, tr, c)
    ot, oc = _popcount(bt), _popcount(bc)
    inter = _popcount(bt[:, None, :] & bc[None, :, :])
    live = (ot[:, None] > 0) & (oc[None, :] > 0) & (t[:, None] != c[None, :])
    ratio = inter / np.maximum(np.maximum(ot[:, None], oc[None, :]), 1)
    return int((live & (ratio < 0.25)).sum()), int((live & (ratio >= 0.25)).sum()), int(max(ot.max(), oc.max()))


def inbound_cases(fx, mask, rng):
    ids_lo, _, fr, tr = G.links(fx, mask)
    n = len(ids_lo)
    r = lambda i: G.rank_of(fx, mask, i)
    hubs = [r(i) for i in range(8, G.HUB + 1)] + [r(G.WIDE0 + k) for k in range(0, G.N_WIDE, 3)]
    halves = [r(9), r(G.POOL), r(16), r(G.POOL + 1), r(G.CHAIN0 + 5), r(G.POOL + 2), r(G.OUT_HUB), r(G.POOL + 3)]
    selfers = [r(G.CHAIN0 + 12), r(G.CHAIN0 + 3), r(G.HUB), r(G.CHAIN0 + 13)]
    indeg = np.bincount(tr, minlength=n)
    popular = np.argsort(-indeg, kind="stable")[:400]
    mid = rng.choice(np.flatnonzero((indeg >= 3) & (indeg <= 40)), 200, replace=False)

    def targets(k):
        base = list(hubs[:6]) + halves[::2] + selfers[:2] + [NO_RANK]
        base += list(rng.choice(popular, 40, replace=False)) + list(rng.choice(mid, 40, replace=False))
        t = np.array(base[:k] + list(rng.choice(base, max(0, k - len(base)))), np.uint32)
        if k >= 3:
            t[k - 1] = t[0]                        # duplicated target
        return t
    t129 = targets(129)
    cand = np.array(list(hubs) + halves[1::2] + halves[::2] + selfers + [NO_RANK] + list(t129[60:75])   # targets of a later pass
                    + list(rng.choice(popular, 40, replace=False)) + list(rng.choice(mid, 60, replace=False)) + list(rng.choice(n, 30, replace=False)),
                    np.uint32)
    cases = []
    for nl, nd in ((1, 0), (0, 1), (32, 32), (33, 32), (64, 0), (64, 65), (65, 64), (129, 0), (0, 129)):
        li, di = targets(nl) if nl != 129 else t129, targets(nd)
        cases.append((li, di, cand, (nl + nd) % 2 == 1, 1.0 if nl % 2 == 0 else 0.25))
    cases.append((np.zeros(0, np.uint32), targets(65), cand, True, 1.0))     # normalized with 0 liked
    return cases


def check_inbound_similarity(fx, mask, rng=None):
    rng = np.random.default_rng(8) if rng is None else rng
    ids_lo, ids_hi, fr, tr = G.links(fx, mask)
    cases = inbound_cases(fx, mask, rng)
    dg = DeviceGraph(_webgraph(fx), skipped_rel=mask)
    try:
        for li, di, ca, norm, ss in cases:
            want = oracle.inbound_similarity(ids_lo, ids_hi, fr, tr, li, di, ca, norm, ss)
            got = dg.inbound_similarity([_id(ids_lo, ids_hi, x) for x in li], [_id(ids_lo, ids_hi, x) for x in di],
                                        [_id(ids_lo, ids_hi, x) for x in ca], norm, ss)
            bad = np.flatnonzero(got.view(np.uint64) != want.view(np.uint64))
            assert bad.size == 0, (len(li), len(di), norm, [(int(i), float(got[i]), float(want[i])) for i in bad[:5]])
    finally:
        dg.close()
    targets = np.concatenate([np.concatenate([li, di]) for li, di, _, _, _ in cases])
    rejected, accepted, most = _prefilter_counts(ids_lo, fr, tr, targets, cases[0][2])
    # word = hash % 16 and bit = hash % 64 share their low four bits, so a word holds at most 4 of its 64 bits: a
    # saturated filter has 64 ones (the hubs')
    assert most == 64
    assert rejected > 100 and accepted > 100, (rejected, accepted)


@pytest.mark.parametrize("mask", [0, SKIPPED_REL])
def test_inbound_similarity_range_graph(mask):
    check_inbound_similarity(G.range_graph(1, "full"), mask)
