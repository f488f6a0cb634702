"""Graph fixtures built to reach the structural edges of the HyperBall and graph-search kernels on purpose (test
infrastructure).

The staging (graph_stage.cu) sorts rows by in-degree and picks the kernel per row: rows of <= QUAD_MAX_DEG (32) in-edges
go to the quad kernels, longer rows are cut into work items of CHUNK_EDGES (1024) edges, and rows of more than one item
park partial maxima that k_pull_merge reduces (one warp per row, eight rows per CTA; each quad of the warp walks the
items i0 + q, i0 + q + 8, ...).  The graph searches (graph_bfs.cu) use the same items.  A random graph reaches these
edges only by chance, so `range_graph` builds rows of exactly the lengths around each boundary and `self_check` proves,
from the oracle's own link derivation, that every one of them is there.

`range_graph(seed, scale)`: SoA edge stream (as synth returns it) over N nodes, N % 32 == 31 (the last bitmap word is
partial), whose kept, de-duplicated, self-loop-free in-degrees -- under both the HyperBall skip mask and mask 0 --
include each of EXACT_DEGREES, one hub of `hub` in-edges, at least 40 rows of 1025..1100 in-edges, and a source with
`out_hub` out-edges; plus NOFOLLOW-first and clean-first duplicates, self-links (one whose first occurrence is skipped),
nodes that occur only on skipped edges, nodes with out-edges only, a 20-node chain, and u128 ids that are all ones or
share a low or a high half with another node.

`chain_graph(length)`: a path of `length` nodes hanging off a dense core of 12 nodes: HyperBall runs more than 256
iterations on it and a breadth-first search from the core meets the 254-level cap of u8 distances."""
import functools

import numpy as np

import oracle
from stract_b200 import synth
from stract_b200.webgraph import RelFlags, SKIPPED_REL

QUAD_MAX_DEG = 32     # graph.cuh
CHUNK_EDGES = 1024    # graph.cuh
MERGE_ROWS_PER_CTA = 8
EXACT_DEGREES = (1, 2, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025, 2047, 2048, 2049, 8192, 8193, 16385)
M64 = (1 << 64) - 1
ALL_ONES = (1 << 128) - 1

# "reduced" keeps every boundary and shrinks only the hub, the out-hub and the node count (the CPU emulator's size)
SCALES = {"full": dict(nodes=(1 << 17) - 1, hub=70_000, out_hub=70_000),
          "reduced": dict(nodes=(1 << 15) - 1, hub=11_900, out_hub=12_000)}

# node indices of the rows built on purpose; the pool (background nodes) starts at POOL
HUB = len(EXACT_DEGREES)            # 17
OUT_HUB = HUB + 1                   # 18
WIDE0, N_WIDE = 19, 40              # rows of 1025..1095 clean in-edges (+ NOFOLLOW-first duplicates: <= 1100 under mask 0)
CHAIN0, CHAIN_LEN = 60, 20
SKIPPED_ONLY0, N_SKIPPED_ONLY = 80, 6
POOL = 100
NOFOLLOW_FIRST_HUB = 300            # extra sources of the hub whose link's first occurrence is NOFOLLOW
NOFOLLOW_FIRST_WIDE = 5             # the same, per wide row


def _ids(n, seed):
    lo, hi = synth.node_ids(np.arange(n, dtype=np.uint64), id_seed=1000 + seed)
    lo = lo.copy(); hi = hi.copy()

    def put(i, v):
        lo[i] = np.uint64(v & M64); hi[i] = np.uint64(v >> 64)
    put(HUB, ALL_ONES)                                   # the hash set's sentinel, on the largest row
    put(POOL + 0, (int(hi[POOL + 0]) << 64) | int(lo[9]))         # shares the low half of the 1023 row
    put(POOL + 1, (int(hi[16]) << 64) | int(lo[POOL + 1]))        # shares the high half of the 16385 row
    put(POOL + 2, (int(hi[POOL + 2]) << 64) | int(lo[CHAIN0 + 5]))   # shares the low half of a chain node
    put(POOL + 3, (int(hi[POOL + 3]) << 64) | int(lo[OUT_HUB]))   # shares the low half of the out-hub
    put(POOL + 4, M64)                                   # hi = 0, lo = all ones
    put(POOL + 5, M64 << 64)                             # hi = all ones, lo = 0
    assert len(set(zip(lo.tolist(), hi.tolist()))) == n
    return lo, hi


@functools.lru_cache(maxsize=4)
def range_graph(seed=1, scale="full"):
    sc = SCALES[scale]
    n, hub, out_hub = sc["nodes"], sc["hub"], sc["out_hub"]
    rng = np.random.default_rng(seed)
    pool = np.arange(POOL, n)
    f, t, r = [], [], []

    def add(src, dst, rel=0):
        src = np.atleast_1d(np.asarray(src, np.int64)); dst = np.broadcast_to(np.asarray(dst, np.int64), src.shape)
        f.append(src); t.append(dst.copy()); r.append(np.full(src.shape, rel, np.int64))
    # rows of exact length: distinct pool sources
    for i, d in enumerate(EXACT_DEGREES):
        add(rng.choice(pool, d, replace=False), i)
    hub_src = rng.choice(pool, hub + NOFOLLOW_FIRST_HUB, replace=False)
    add(hub_src[hub:], HUB, RelFlags.NOFOLLOW)                      # first occurrence skipped: the link is not kept ...
    add(hub_src[:hub], HUB)
    add(hub_src[hub:], HUB)                                         # ... though it comes again clean (first wins)
    for k in range(N_WIDE):
        d = 1025 + (70 * k) // (N_WIDE - 1)
        src = rng.choice(pool, d + NOFOLLOW_FIRST_WIDE, replace=False)
        add(src[d:], WIDE0 + k, RelFlags.NOFOLLOW)
        add(src, WIDE0 + k)
    add(np.full(out_hub, OUT_HUB), rng.choice(pool, out_hub, replace=False))
    # clean-first duplicates (later NOFOLLOW copies change nothing) on exact rows
    for i in (10, 13, 16):
        add(f[i][:50], i, RelFlags.NOFOLLOW)
    # a chain fed from the pool
    add(pool[7], CHAIN0)
    for k in range(CHAIN_LEN - 1):
        add(CHAIN0 + k, CHAIN0 + k + 1)
    # self-links: on hubs, on chain nodes, and one whose first occurrence is skipped
    add([HUB, 16, 15], [HUB, 16, 15])
    add([CHAIN0 + 3, CHAIN0 + 9], [CHAIN0 + 3, CHAIN0 + 9])
    add(CHAIN0 + 12, CHAIN0 + 12, RelFlags.NOFOLLOW)
    add(CHAIN0 + 12, CHAIN0 + 12)
    add(HUB, HUB, RelFlags.NOFOLLOW)
    # nodes that occur only on skipped edges (kept under mask 0: one in-edge and one out-edge each)
    so = np.arange(SKIPPED_ONLY0, SKIPPED_ONLY0 + N_SKIPPED_ONLY)
    add(so, rng.choice(pool, so.size), RelFlags.NOFOLLOW)
    add(rng.choice(pool, so.size), so, RelFlags.NOFOLLOW | RelFlags.TAG)
    # background: every other node links to two pool nodes (10 % NOFOLLOW); pool nodes nobody picks have out-edges only
    others = np.setdiff1d(np.arange(n), np.append(so, OUT_HUB))
    src = np.repeat(others, 2)
    dst = rng.choice(pool, src.size)
    add(src, dst)
    r[-1] = np.where(rng.random(src.size) < 0.1, RelFlags.NOFOLLOW, 0).astype(np.int64)
    fi = np.concatenate(f); ti = np.concatenate(t); rel = np.concatenate(r).astype(np.uint64)
    lo, hi = _ids(n, seed)
    d = dict(from_lo=lo[fi], from_hi=hi[fi], to_lo=lo[ti], to_hi=hi[ti], rel_flags=rel)
    return dict(arrays=d, n=n, hub=hub, out_hub=out_hub, seed=seed, scale=scale, index_lo=lo, index_hi=hi)


@functools.lru_cache(maxsize=2)
def chain_graph(length=300, seed=3):
    """core (12 nodes, every ordered pair linked) -> c0 -> c1 -> ... -> c(length-1); c0 also links back into the core and
    every tenth chain node has a self-link (the first one skipped first, then clean)."""
    core = 12
    f, t, r = [], [], []
    for a in range(core):
        for b in range(core):
            if a != b:
                f.append(a); t.append(b); r.append(0)
    prev = 0
    for k in range(length):
        f.append(prev); t.append(core + k); r.append(0)
        prev = core + k
    f.append(core); t.append(1); r.append(0)
    for k in range(0, length, 10):
        if k == 10:
            f.append(core + k); t.append(core + k); r.append(RelFlags.NOFOLLOW)
        f.append(core + k); t.append(core + k); r.append(0)
    lo, hi = synth.node_ids(np.arange(core + length, dtype=np.uint64), id_seed=2000 + seed)
    fi = np.array(f); ti = np.array(t)
    d = dict(from_lo=lo[fi], from_hi=hi[fi], to_lo=lo[ti], to_hi=hi[ti], rel_flags=np.array(r, np.uint64))
    return dict(arrays=d, n=core + length, core=core, length=length, index_lo=lo, index_hi=hi)


def args(fx):
    d = fx["arrays"]
    return d["from_lo"], d["from_hi"], d["to_lo"], d["to_hi"], d["rel_flags"]


@functools.lru_cache(maxsize=8)
def _links(key, mask):
    fx = range_graph(*key) if key[0] != "chain" else chain_graph(*key[1:])
    return oracle.graph_links(*args(fx), skip_mask=mask)


def links(fx, mask):
    """(ids_lo, ids_hi, from_rank, to_rank) of the kept links (self-links included), cached per fixture and mask."""
    key = ("chain", fx["length"]) if "length" in fx else (fx["seed"], fx["scale"])
    return _links(key, int(mask))


def rank_of(fx, mask, idx):
    """rank (position in ascending id order) of fixture node index `idx`"""
    ids_lo, ids_hi, _, _ = links(fx, mask)
    lo, hi = int(fx["index_lo"][idx]), int(fx["index_hi"][idx])
    key = ids_hi.astype(object) * (1 << 64) + ids_lo.astype(object)
    r = int(np.searchsorted(key, (hi << 64) | lo))
    assert key[r] == (hi << 64) | lo
    return r


def structure(fx, mask):
    """in-degree / out-degree of every rank over the CSR the staging builds (self-links dropped) and the row classes
    with the staging's rule"""
    ids_lo, _, fr, tr = links(fx, mask)
    n = len(ids_lo)
    keep = fr != tr
    indeg = np.bincount(tr[keep], minlength=n)
    outdeg = np.bincount(fr[keep], minlength=n)
    warp = indeg[indeg > QUAD_MAX_DEG]
    items = -(-warp // CHUNK_EDGES)
    return dict(n=n, indeg=indeg, outdeg=outdeg, warp_rows=int(warp.size), multi_rows=int((warp > CHUNK_EDGES).sum()),
                items=int(items.sum()), max_items=int(items.max()) if items.size else 0, looping_merge_rows=int((items > 8).sum()))


def self_check(fx, mask=SKIPPED_REL):
    """Every boundary of range_graph is in the kept links of this mask (a generator change cannot drop one quietly)."""
    s = structure(fx, mask)
    n, indeg, outdeg = s["n"], s["indeg"], s["outdeg"]
    assert n == fx["n"] and n % 32 == 31, n
    present = set(np.unique(indeg).tolist())
    missing = [d for d in EXACT_DEGREES if d not in present]
    assert not missing, missing
    hub_rank = rank_of(fx, mask, HUB)
    lo_items = -(-fx["hub"] // CHUNK_EDGES)
    assert -(-int(indeg[hub_rank]) // CHUNK_EDGES) == lo_items, (indeg[hub_rank], fx["hub"])
    assert ((indeg >= 1025) & (indeg <= 1100)).sum() >= 40
    assert outdeg.max() == fx["out_hub"]
    # work items with the staging's rule: more multi-item rows than one k_pull_merge CTA takes, rows whose merge loops
    assert s["multi_rows"] >= 40 + 8 and s["multi_rows"] > MERGE_ROWS_PER_CTA
    assert s["looping_merge_rows"] >= 3 and s["max_items"] == max(lo_items, 17)
    assert s["warp_rows"] > s["multi_rows"] and s["items"] > s["warp_rows"]
    if fx["scale"] == "full":
        assert s["max_items"] == 69
    # duplicates: a NOFOLLOW-first link into the hub is dropped under the HyperBall mask and kept under mask 0
    ids_lo, ids_hi, fr, tr = links(fx, mask)
    want_hub = fx["hub"] + (NOFOLLOW_FIRST_HUB if mask & RelFlags.NOFOLLOW == 0 else 0)
    assert indeg[hub_rank] == want_hub, (indeg[hub_rank], want_hub)
    # self-links: kept ones on the hub and on chain nodes; the skipped-first one only under mask 0
    selfs = set(fr[fr == tr].tolist())
    assert hub_rank in selfs and rank_of(fx, mask, CHAIN0 + 3) in selfs
    assert (rank_of(fx, mask, CHAIN0 + 12) in selfs) == (mask & RelFlags.NOFOLLOW == 0)
    # nodes only on skipped edges are isolated under the HyperBall mask; nodes with out-edges only exist
    so = [rank_of(fx, mask, SKIPPED_ONLY0 + k) for k in range(N_SKIPPED_ONLY)]
    if mask & RelFlags.NOFOLLOW:
        assert all(indeg[r] == 0 and outdeg[r] == 0 for r in so)
    assert ((indeg == 0) & (outdeg > 0)).sum() > 100
    # ids: the all-ones id (last rank), shared low halves and shared high halves
    assert int(ids_lo[-1]) == M64 and int(ids_hi[-1]) == M64 and hub_rank == n - 1
    assert np.unique(ids_lo).size < n and np.unique(ids_hi).size < n
    assert (ids_hi == 0).any() and (ids_lo == 0).any()
    return s
