"""Posting lists that reach the edges of tantivy's posting format on purpose (no pytest import): full blocks whose doc-delta
and tf widths are chosen one by one (0..31 / 0..32 bits), VInt tails with 1- to 5-byte doc gaps and tfs, block-wand tf
codes 254 / 255 (saturated) on short documents, every fieldnorm code on a posted document, and doc ids up to max_doc - 1
next to TERMINATED.  Each block of a width term carries ONE posting of the target width and 127 small ones: a mask or
word-straddle error then corrupts small values, whose scores visibly change (an f32 BM25 score hides tf errors above ~4 000).

`range_index` parses the skip entries and tails it wrote and asserts that every target was produced, so a change to the
generator cannot silently shrink what the tests cover."""
import numpy as np

WD = (0, 1, 7, 8, 9, 15, 16, 17, 24, 31)
WT = (0, 1, 4, 5, 8, 9, 12, 16, 17, 24, 31, 32)
DFS = (1, 127, 128, 129, 255, 256, 257)
SATURATED = (254, 255, 256, 300, 5000, 10 ** 6, 10 ** 8)   # best tf of consecutive blocks: codes 254, 255, then saturated
BIG_DF = 70_000                                            # one clause above 65 536 postings: k_topk_warp<AND>
TF_WIDE_MAX = 3 << 30                                      # tf - 1 ceiling: a record-2 block's u32 tf sum stays < 2^32


def _wide(rng, w, hi):
    """a value of exactly w bits, at most hi"""
    if w == 0:
        return 0
    lo, top = 1 << (w - 1), min((1 << w) - 1, hi)
    assert top >= lo, (w, hi)
    return int(rng.integers(lo, top + 1))


def _small(rng, w, n):
    return rng.integers(0, 1 << min(w, 3), n, dtype=np.int64)


def _block(rng, prev, wd, wt, room):
    """128 postings after doc `prev`: deltas - 1 and tfs - 1 of widths exactly wd / wt (one wide value each, at a random
    slot; the others < 8).  `room` bounds the doc span."""
    dm1 = _small(rng, wd, 128)
    # a 24 / 31-bit jump takes at most a quarter of the room above its minimum: the tail after it keeps room for 5-byte gaps
    hi = (1 << wd) - 1 if wd < 24 else (1 << (wd - 1)) + max(room - 1024 - (1 << (wd - 1)), 0) // 4
    dm1[int(rng.integers(0, 128))] = _wide(rng, wd, hi)
    tm1 = _small(rng, wt, 128)
    tm1[int(rng.integers(0, 128))] = _wide(rng, wt, TF_WIDE_MAX)
    docs = prev + np.cumsum(dm1 + 1)
    return docs, tm1 + 1


def _tail(rng, prev, gap_bytes, tf_bytes, n, room):
    """n VInt-tail postings after doc `prev`: one gap (tf) of each requested VInt length, the rest small"""
    gaps = rng.integers(1, 4, n, dtype=np.int64)
    tfs = rng.integers(1, 9, n, dtype=np.int64)
    slots = rng.permutation(n)
    for i, b in enumerate(gap_bytes):
        lo = 1 << (7 * (b - 1)) if b > 1 else 1
        hi = min((1 << (7 * b)) - 1, room - 4 * n)
        assert hi >= lo, (b, room)
        gaps[slots[i]] = int(rng.integers(lo, hi + 1))
        room -= int(gaps[slots[i]])
    for i, b in enumerate(tf_bytes):
        tfs[slots[-1 - i]] = int(rng.integers(1 << (7 * (b - 1)) if b > 1 else 1, min((1 << (7 * b)) - 1, 0xFFFFFFFF) + 1))
    return prev + np.cumsum(gaps), tfs


def _width_term(rng, base, specs, tail_n, gap_bytes, tf_bytes, limit):
    """a lead block from `base`, one block per (wd, wt) spec, then a VInt tail; every doc < limit"""
    d0 = base + np.cumsum(rng.integers(1, 5, 128)) - 1
    docs, tfs = [d0], [rng.integers(1, 9, 128)]
    prev = int(d0[-1])
    for wd, wt in specs:
        d, t = _block(rng, prev, wd, wt, limit - prev)
        docs.append(d); tfs.append(t); prev = int(d[-1])
    if tail_n:
        d, t = _tail(rng, prev, gap_bytes, tf_bytes, tail_n, limit - 1 - prev)
        docs.append(d); tfs.append(t)
    docs = np.concatenate(docs); tfs = np.concatenate(tfs)
    assert docs[-1] < limit and np.all(np.diff(docs) > 0) and tfs.max() <= 0xFFFFFFFF
    return docs.astype(np.uint32), tfs.astype(np.uint32)


def _subset(rng, docs, frac, extra_tf_bytes=()):
    keep = np.sort(rng.choice(docs.size, max(1, int(docs.size * frac)), replace=False))
    tfs = rng.integers(1, 9, keep.size, dtype=np.int64)
    for i, b in enumerate(extra_tf_bytes):
        tfs[int(rng.integers(0, keep.size))] = 1 << (7 * (b - 1))
    return docs[keep].astype(np.uint32), tfs.astype(np.uint32)


def range_index(seed, max_doc, record_option=1, big=True):
    """The terms (docs, tfs) and the fieldnorm ids of an index over [0, max_doc) that reaches every width the doc space
    allows.  Returns a dict: docs, tfs (lists), ids (u8[max_doc]), groups (lists of term ordinals whose doc sets overlap:
    AND queries draw from one group), saturated (ordinals of the block-wand saturation terms), tail_max (a term whose best
    doc sits in its tail behind full-block postings above max_score), targets (what the self-check demands)."""
    rng = np.random.default_rng(seed)
    limit = max_doc
    wds = [w for w in WD if (w < 24 or (1 << (w - 1)) + 4096 < limit // 2)]
    td, tt, groups = [], [], []

    def add(d, t):
        td.append(d); tt.append(t)
        return len(td) - 1

    tail_gaps = [b for b in (1, 2, 3, 4, 5) if (1 << (7 * (b - 1))) * 3 < limit]
    for wd in wds:
        # one block per tf width; a 24 / 31-bit jump uses a large part of the doc space: one such block per term then
        per_term = [[(wd, wt) for wt in WT]] if wd < 24 else [[(wd, wt)] for wt in WT]
        for specs in per_term:
            span = sum(1 << w for w, _ in specs if w < 24) + 600 * len(specs) + 1024
            if wd >= 24:
                base = int(rng.integers(0, 1 << 16))
            else:
                base = int(rng.integers(0, max(limit - span - (4 << (7 * (tail_gaps[-1] - 1))), 1)))   # room for the tail gaps
            tail_n = int(rng.integers(10, 128))
            d, t = _width_term(rng, base, specs, tail_n, tail_gaps if wd < 24 else tail_gaps[-1:], (1, 2, 3, 4, 5), limit)
            x = add(d, t)
            # overlapping partners for AND: two halves of the term and a quarter with wide tfs
            groups.append([x, add(*_subset(rng, d, 0.5)), add(*_subset(rng, d, 0.5)), add(*_subset(rng, d, 0.25, (3, 4, 5)))])
    # doc_freqs on both sides of the block size, as subsets of one width term (a group of their own)
    src = td[groups[len(groups) // 2][0]]
    g = []
    for df in DFS:
        keep = np.sort(rng.choice(src.size, df, replace=False))
        g.append(add(src[keep], rng.integers(1, 9, df).astype(np.uint32)))
    groups.append(g + [groups[len(groups) // 2][0]])
    # a tail that ends at max_doc - 1 (next to TERMINATED) and a full block that does
    d = np.arange(limit - 1 - 129 * 3, limit, 3, dtype=np.int64)[-129:]
    nb = add(d.astype(np.uint32), rng.integers(1, 9, d.size).astype(np.uint32))
    d = np.arange(limit - 128, limit, dtype=np.int64)
    ne = add(d.astype(np.uint32), rng.integers(1, 9, 128).astype(np.uint32))
    groups.append([nb, ne])
    # block-wand saturation: each block's best posting is a large tf on a doc with fieldnorm id 0; later blocks score higher
    short = []
    base = int(rng.integers(0, limit // 2))
    d = base + np.cumsum(rng.integers(1, 5, 128 * len(SATURATED) + 40))
    t = rng.integers(1, 9, d.size)
    for b, tf in enumerate(SATURATED):
        i = b * 128 + int(rng.integers(0, 128))
        t[i] = tf; short.append(int(d[i]))
    s0 = add(d.astype(np.uint32), t.astype(np.uint32))
    s1 = add(*_subset(rng, td[s0], 0.5))
    groups.append([s0, s1])
    saturated = [s0]
    # the best doc in a VInt tail behind six full-block postings that score above Bm25Weight::max_score: a one-clause
    # block-wand walk (block_wand_single_scorer) bounds the tail it has not loaded by max_score and skips it at k <= 6
    base = int(rng.integers(0, limit // 2))
    d = base + 3 * np.arange(276)
    t = rng.integers(1, 9, d.size)
    for j, i in enumerate((5, 60, 120, 130, 200, 250)):
        t[i] = 100_000 + 1000 * j; short.append(int(d[i]))
    t[262] = 10 ** 7; short.append(int(d[262]))
    tail_max = [add(d.astype(np.uint32), t.astype(np.uint32))]
    groups.append(tail_max)
    if big:   # > 65 536 postings, wide blocks sprinkled in
        base = int(rng.integers(0, limit // 4))
        specs = [(17 if limit > 1 << 22 else 9, WT[i % len(WT)]) if i % 40 == 0 else (2, 2) for i in range(BIG_DF // 128 - 1)]
        d, t = _width_term(rng, base, specs, BIG_DF % 128, (1, 2), (1, 2, 3), limit)
        assert d.size > 65_536
        x = add(d, t)
        groups.append([x, add(*_subset(rng, d, 0.3)), add(*_subset(rng, d, 0.02))])
    # fieldnorm ids: a repeated LogNormal pattern; every code on a posted doc; the saturation docs are the shortest
    pat = np.searchsorted(_table(), np.maximum(1, rng.lognormal(4.0, 0.8, 1 << 20)).astype(np.uint32), side="right") - 1
    ids = np.resize(pat.astype(np.uint8), limit)
    posted = np.unique(np.concatenate([x[:: max(1, x.size // 64)] for x in td]))
    posted = posted[~np.isin(posted, short)]
    ids[rng.choice(posted, 256, replace=False)] = np.arange(256, dtype=np.uint8)
    ids[short] = 0
    targets = {"wd": set(wds), "wt": set(WT), "pairs": {(8, 8), (8, 9), (16, 0), (0, 16), (16, 1)},
               "gap_bytes": set(tail_gaps) | {1}, "tf_bytes": {1, 2, 3, 4, 5}, "bw_tf": {254, 255},
               "dfs": set(DFS) | ({BIG_DF} if big else set())}
    return {"docs": td, "tfs": tt, "ids": ids, "max_doc": limit, "groups": groups, "saturated": saturated, "tail_max": tail_max,
            "record_option": record_option, "targets": targets}


def _table():
    from stract_b200.bm25 import fieldnorm_table
    return fieldnorm_table()


def parse_term(data, off, ln, df, record_option):
    """skip entries and tail VInt lengths of one term: dict of db, tb (lists), bw_id, bw_tf, gap_bytes, tf_bytes"""
    b = data[int(off):int(off) + int(ln)].tobytes()
    nfull, p = df // 128, 0
    out = {"db": [], "tb": [], "bw_id": [], "bw_tf": [], "gap_bytes": [], "tf_bytes": []}
    body = 0
    if df >= 128:
        skip_len, sh = 0, 0
        while True:
            x = b[p]; p += 1
            skip_len |= (x & 127) << sh
            if x & 128:
                break
            sh += 7
        stride = 12 if record_option == 2 else 8
        assert skip_len == nfull * stride
        for j in range(nfull):
            e = b[p + j * stride:p + (j + 1) * stride]
            assert e[4] & 0x40
            out["db"].append(e[4] & 0x3F); out["tb"].append(e[5])
            out["bw_id"].append(e[stride - 2]); out["bw_tf"].append(e[stride - 1])
            body += (out["db"][-1] + out["tb"][-1]) * 16
        p += skip_len
    p += body
    lens = []
    for _ in range(2 * (df - nfull * 128)):
        n = 1
        while not b[p] & 0x80:
            p += 1; n += 1
        p += 1; lens.append(n)
    assert p == len(b), (p, len(b))
    half = len(lens) // 2
    out["gap_bytes"], out["tf_bytes"] = lens[:half], lens[half:]
    return out


def self_check(fx, data, term_infos):
    """every target width / code / VInt length / doc_freq was produced, every fieldnorm code sits on a posted doc;
    `term_infos` = (postings_off, postings_len, doc_freq) arrays.  Returns what was produced."""
    off, ln, dfs = term_infos
    got = {"wd": set(), "wt": set(), "pairs": set(), "gap_bytes": set(), "tf_bytes": set(), "bw_tf": set(), "dfs": set()}
    staged = direct = 0
    for t in range(len(fx["docs"])):
        df = int(dfs[t])
        r = parse_term(data, off[t], ln[t], df, fx["record_option"])
        got["wd"] |= set(r["db"]); got["wt"] |= set(r["tb"]); got["pairs"] |= set(zip(r["db"], r["tb"]))
        got["gap_bytes"] |= set(r["gap_bytes"]); got["tf_bytes"] |= set(r["tf_bytes"]); got["bw_tf"] |= set(r["bw_tf"])
        got["dfs"].add(df)
        staged += sum(0 < (a + c) * 16 <= 256 for a, c in zip(r["db"], r["tb"]))
        direct += sum((a + c) * 16 > 256 for a, c in zip(r["db"], r["tb"]))
    for k, want in fx["targets"].items():
        assert want <= got[k], (k, sorted(want - got[k]))
    assert staged and direct, "k_or3: blocks on both sides of the staging limit"
    posted = np.unique(np.concatenate(fx["docs"]))
    assert np.unique(fx["ids"][posted]).size == 256, "every fieldnorm code on a posted doc"
    assert int(posted[-1]) == fx["max_doc"] - 1
    return got


PW = (0, 1, 2, 7, 8, 9, 15, 16, 17, 24, 31)   # position-delta block widths
TF16 = 1 << 16                                # a posting tf of 17 bits (tf - 1 of width 16) in a full block


def positions_index(seed, n_docs=4096):
    """A record-option-2 index given as per-doc position arrays (the form of phrase_fixtures.make_segment).  Term 0: one
    full positions block per width in PW, each with one delta of that width and 127 small ones, and a VInt tail with
    1- to 5-byte deltas (up to 2^31 - 1).  Postings never straddle a block, so a position stays below 2^32.  Term 1: a
    doc with tf 2^16 + 1 (longer than the phrase kernels' shared-memory buffer) among 127 others in a full block.
    Returns (index, deltas): deltas[t] = the term's whole position-delta stream, as the `.pos` file stores it."""
    from stract_b200.bm25 import fieldnorm_table
    rng = np.random.default_rng(seed)
    streams = []        # per posting: its deltas
    for w in PW:
        if w == 0:      # every delta 0: 128 postings of tf 1 at position 0
            streams += [np.zeros(1, np.int64)] * 128
            continue
        dl = rng.integers(1, min(1 << w, 8), 128, dtype=np.int64)
        dl[int(rng.integers(0, 128))] = _wide(rng, w, (1 << 31) - 1)
        cuts = np.sort(rng.choice(np.arange(1, 128), 12, replace=False))
        streams += np.split(dl, cuts)
    for b in (1, 2, 3, 4, 5):   # the tail: each wide value opens a posting of its own
        lo = 1 << (7 * (b - 1)) if b > 1 else 1
        streams.append(np.array([int(rng.integers(lo, min((1 << (7 * b)) - 1, (1 << 31) - 1) + 1))] + list(rng.integers(1, 8, 2))))
    assert sum(s.size for s in streams) % 128 != 0
    t0_docs = np.sort(rng.choice(n_docs, len(streams), replace=False)).astype(np.uint32)
    t0_pos = [np.cumsum(s).astype(np.uint32) for s in streams]
    assert all(int(np.cumsum(s)[-1]) < 1 << 32 for s in streams)
    tfs1 = rng.integers(1, 4, 130)
    tfs1[int(rng.integers(0, 128))] = TF16 + 1
    t1_docs = np.sort(rng.choice(n_docs, tfs1.size, replace=False)).astype(np.uint32)
    t1_pos = [np.sort(rng.choice(1 << 20, int(tf), replace=False)).astype(np.uint32) for tf in tfs1]
    terms = [{"docs": t0_docs, "positions": t0_pos}, {"docs": t1_docs, "positions": t1_pos}]
    ids = rng.integers(0, 256, n_docs).astype(np.uint8)
    total = int(fieldnorm_table()[ids].astype(np.uint64).sum())
    deltas = [np.concatenate([np.diff(p, prepend=np.uint32(0)).astype(np.uint32) for p in t["positions"]]) for t in terms]
    return {"fieldnorm_ids": ids, "terms": terms, "total_num_tokens": total}, deltas


def parse_positions(data, off, ln):
    """block widths and tail VInt lengths of one term's positions: [VInt n_blocks][width per block][blocks][tail]"""
    b = data[int(off):int(off) + int(ln)].tobytes()
    n, sh, p = 0, 0, 0
    while True:
        x = b[p]; p += 1
        n |= (x & 127) << sh
        if x & 128:
            break
        sh += 7
    widths = list(b[p:p + n])
    p += n + sum(w * 16 for w in widths)
    lens = []
    while p < len(b):
        m = 1
        while not b[p] & 0x80:
            p += 1; m += 1
        p += 1; lens.append(m)
    return widths, lens
