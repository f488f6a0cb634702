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


# ---- positional fixtures: phrases, optic patterns and term distances at wide positions ------------------------------------
TOP = 0xFFFFFFFF


def _anchor_streams(rng):
    """The anchor's postings as position arrays: one full positions block per width in PW (one delta of that width, 127
    small ones, split into ~13 postings that never straddle a block), a block of width 32 whose postings all start at or
    above 2^31, then a VInt tail whose deltas take 1 to 5 bytes"""
    streams = []
    for w in PW:
        if w == 0:      # every delta 0: 128 postings of tf 1 at position 0
            streams += [np.zeros(1, np.int64)] * 128
            continue
        dl = rng.integers(1, min(1 << w, 8), 128, dtype=np.int64)
        dl[int(rng.integers(0, 128))] = _wide(rng, w, (1 << 31) - 1)
        streams += np.split(dl, np.sort(rng.choice(np.arange(1, 128), 12, replace=False)))
    dl = rng.integers(1, 8, 128, dtype=np.int64)
    cuts = np.arange(0, 128, 16)
    dl[cuts] = (1 << 31) + rng.integers(0, 1 << 29, cuts.size)      # 8 postings of 16 positions from 2^31 up
    streams += np.split(dl, cuts[1:])
    for b in (1, 2, 3, 4, 5):   # the tail: each wide value opens a posting of its own
        lo = 1 << (7 * (b - 1)) if b > 1 else 1
        streams.append(np.array([int(rng.integers(lo, min((1 << (7 * b)) - 1, (1 << 31) - 1) + 1))] + list(rng.integers(1, 8, 2))))
    pos = [np.cumsum(s) for s in streams]
    assert all(int(p[-1]) < 1 << 32 for p in pos) and sum(p.size for p in pos) % 128 != 0
    return [p.astype(np.uint32) for p in pos]


def _spread_docs(rng, n, max_doc):
    """n ascending doc ids over [0, max_doc): a dense run, a jump of about max_doc / 2 inside the first block, random
    docs above it, and max_doc - 1 last"""
    a = n // 3
    dense = np.arange(a, dtype=np.int64) * 3
    rest = np.sort(rng.choice(np.arange(max_doc // 2, max_doc - 1, dtype=np.int64), n - a - 1, replace=False))
    return np.concatenate([dense, rest, [max_doc - 1]]).astype(np.uint32)


def _partner(rng, docs, pos, keep, shift, frac=1.0):
    """a term on the anchor's documents `keep` (indices), at the anchor's positions + shift (an int or a per-position
    array drawer), on a fraction of the positions (at least one)"""
    d, p = [], []
    for i in keep:
        x = pos[i].astype(np.int64)
        if frac < 1.0:
            x = x[np.sort(rng.choice(x.size, max(1, int(x.size * frac)), replace=False))]
        s = shift(x.size) if callable(shift) else shift
        y = np.unique(x + s)
        d.append(docs[i]); p.append(y.astype(np.uint32))
    return {"docs": np.array(d, np.uint32), "positions": p}


def positional_range_index(seed, max_doc):
    """A record-option-2 index over [0, max_doc) given as per-document positions (the form of
    phrase_fixtures.make_segment).  Term roles (fx["roles"]):
      anchor     one positions block per delta width in PW and one of width 32 (positions from 2^31 up), a VInt tail with
                 1- to 5-byte deltas; its doc ids take wide doc deltas and end at max_doc - 1
      plus1/2    the anchor's positions + 1 / + 2 on a subset of its postings: slop-0 phrases match at wide positions
      near1..3   the anchor's positions + 1..3 (random per position): slop 1..3
      df128 .. df257, vint   the anchor's positions + 1 on 128, 129, 256, 257 and 40 (VInt tail only) postings
      wrap_a/b/c on documents where the anchor sits at position 0: wrap_a at 0, wrap_b at 4, wrap_c at 2^32 - 1.  The
                 phrase (wrap_a, wrap_b, wrap_c) with offsets (0, 1, 2) and slop >= 3 carries slop 3 from the first pair
                 into `3 + abs_diff(2, 2^32 - 1)`, which wraps to 0 in u32: it matches only because the sum wraps
      big_a/b    one posting of tf 2^16 + 1 (among 127 others in a full block) and the same positions + 1: a verify pass
                 over global scratch
    `counted` = (docs, token counts) of the documents with positions (token_counts makes the dense column): it puts
    num_tokens - 1 on the anchor's last position for its postings above 2^30 (end anchors at wide positions) and above
    every position elsewhere.  Memory stays sparse up to max_doc = 2^31 - 2."""
    from stract_b200.bm25 import fieldnorm_table
    rng = np.random.default_rng(seed)
    apos = _anchor_streams(rng)
    adocs = _spread_docs(rng, len(apos), max_doc)
    terms, roles = [{"docs": adocs, "positions": apos}], {"anchor": 0}

    def add(name, t):
        roles[name] = len(terms); terms.append(t)

    na = len(apos)
    sub = lambda n: np.sort(rng.choice(na, n, replace=False))
    add("plus1", _partner(rng, adocs, apos, sub(int(na * 0.7)), 1, 0.8))
    add("plus2", _partner(rng, adocs, apos, sub(int(na * 0.6)), 2, 0.8))
    for s in (1, 2, 3):
        add(f"near{s}", _partner(rng, adocs, apos, sub(int(na * 0.5)), lambda n, s=s: rng.integers(1, s + 1, n), 0.7))
    for df in (128, 129, 256, 257, 40):
        add("vint" if df < 128 else f"df{df}", _partner(rng, adocs, apos, sub(df), 1, 0.8))
    zero = [i for i in range(na) if apos[i].size == 1 and apos[i][0] == 0]
    wd = np.sort(rng.choice(zero, 12, replace=False))
    one = lambda idx, p: {"docs": adocs[idx], "positions": [np.array([p], np.uint32)] * len(idx)}
    add("wrap_a", one(wd[:6], 0))
    add("wrap_b", one(wd[:8], 4))
    add("wrap_c", one(wd[1:12], TOP))
    # tf 2^16 + 1: the 200th posting of a 300-posting term over the anchor's doc range, and the same positions + 1
    bd = np.sort(rng.choice(max_doc, 300, replace=False)).astype(np.uint32)
    bp = [np.sort(rng.choice(1 << 20, int(rng.integers(1, 4)), replace=False)).astype(np.uint32) for _ in bd]
    bp[200] = np.sort(rng.choice(1 << 24, TF16 + 1, replace=False)).astype(np.uint32)
    add("big_a", {"docs": bd, "positions": bp})
    add("big_b", {"docs": bd[195:205], "positions": [p + 1 for p in bp[195:205]]})
    ids = np.empty(max_doc, np.uint8)
    for a in range(0, max_doc, 1 << 26):
        ids[a:a + (1 << 26)] = rng.integers(0, 256, min(1 << 26, max_doc - a), dtype=np.uint8)
    table = fieldnorm_table().astype(np.uint64)
    total = sum(int(np.bincount(ids[a:a + (1 << 26)], minlength=256) @ table) for a in range(0, max_doc, 1 << 26))
    last = {}
    for t in terms:
        for d, p in zip(t["docs"], t["positions"]):
            last[int(d)] = max(last.get(int(d), 0), int(p[-1]) + 1)
    posted = np.array(sorted(last), np.int64)
    cvals = np.array([last[int(d)] for d in posted], np.uint64) + rng.integers(0, 3, posted.size).astype(np.uint64)
    wide = [i for i in range(na) if int(apos[i][-1]) >= 1 << 30]
    cvals[np.searchsorted(posted, adocs[wide])] = [last[int(d)] for d in adocs[wide]]
    return {"fieldnorm_ids": ids, "terms": terms, "total_num_tokens": total, "roles": roles, "counted": (posted, cvals),
            "max_doc": max_doc, "end_anchored": adocs[wide]}


def token_counts(fx):
    """the dense token-count column of a positional_range_index (one u64 per document; 0 for documents without positions)"""
    c = np.zeros(fx["max_doc"], np.uint64)
    c[fx["counted"][0]] = fx["counted"][1]
    return c


def token_count(fx, d):
    posted, cvals = fx["counted"]
    i = int(np.searchsorted(posted, d))
    return int(cvals[i]) if i < posted.size and posted[i] == d else 0


def positional_self_check(fx):
    """every target of positional_range_index was produced: anchor block widths PW + 32 and 1- to 5-byte tail deltas in the
    `.pos` bytes, doc ids up to max_doc - 1 and wide doc deltas in the postings, the doc_freqs, slop-0 matches at positions
    >= 2^31, the u32 wrap (a match the unwrapped sum would reject), the tf 2^16 + 1 posting, and end-anchored documents
    whose last position is >= 2^30.  Returns the anchor's widths and tail lengths and its largest doc-delta width."""
    import phrase_oracle as O
    from stract_b200.bm25 import encode_positions, encode_postings
    terms, roles = fx["terms"], fx["roles"]
    tfs = [np.array([p.size for p in t["positions"]], np.uint32) for t in terms]
    off = np.concatenate([[0], np.cumsum([t["docs"].size for t in terms])])
    pos, po, pl = encode_positions(np.concatenate([p for t in terms for p in t["positions"]]), np.concatenate(tfs), off)
    widths, lens = parse_positions(pos, po[0], pl[0])
    assert set(widths) == set(PW) | {32} and set(lens) >= {1, 2, 3, 4, 5}, (sorted(set(widths)), sorted(set(lens)))
    data, infos = encode_postings([t["docs"] for t in terms], tfs, fx["fieldnorm_ids"], 1.0, record_option=2)
    a = parse_term(data, infos[0].postings_off, infos[0].postings_len, infos[0].doc_freq, 2)
    assert max(a["db"]) >= (20 if fx["max_doc"] > 1 << 22 else 9), a["db"]
    assert int(max(t["docs"][-1] for t in terms)) == fx["max_doc"] - 1
    dfs = {t["docs"].size for t in terms}
    assert {128, 129, 256, 257} <= dfs and min(dfs) < 128
    assert max(int(t.max()) for t in tfs) == TF16 + 1
    cache = O.tf_cache(np.float32(1.0), np.arange(256))
    idx = {"fieldnorm_ids": fx["fieldnorm_ids"], "terms": terms}
    hits = O.phrase_search(idx, [roles["anchor"], roles["plus1"]], [0, 1], 0, True, np.float32(1.0), cache)
    anchor = terms[roles["anchor"]]
    assert any(int(anchor["positions"][int(np.searchsorted(anchor["docs"], d))][-1]) >= 1 << 31 for _, d in hits)
    wq = [roles["wrap_a"], roles["wrap_b"], roles["wrap_c"]]
    wh = O.phrase_search(idx, wq, [0, 1, 2], 3, True, np.float32(1.0), cache)
    assert wh and all(int(x) == TOP for d in (h[1] for h in wh)
                      for x in terms[wq[2]]["positions"][int(np.searchsorted(terms[wq[2]]["docs"], d))]), "the wrap case"
    ea = fx["end_anchored"]
    assert ea.size and all(token_count(fx, d) - 1 >= 1 << 30 for d in ea)
    return widths, lens, max(a["db"])


HUGE_TF = 1 << 28     # positions per huge posting: 1 GiB of 32-bit deltas each


def huge_positions_term(seed, n_huge=5, late_tfs=(40, 90, 126, 3, 60, 5), max_doc=64):
    """One term whose positions pass 4 GiB of bit-packed data, written straight to bytes.  At bit width 32 a BitPacker4x
    block is its 128 values as little-endian u32 in order, so the `.pos` data of the n_huge postings of tf HUGE_TF is the
    delta array itself: small deltas and one value with bit 31 set per block.  After them come `late_tfs` small postings
    with ordinary deltas, whose full blocks (real widths) start past byte 4 GiB of the term's data; the rest is VInt tail.
    df < 128: the postings are all VInt tail, so no skip entry sums a tf.

    Term 0 is that term (docs 0 .. n_huge-1 huge, then the late docs); term 1 is a partner on the late docs only, at the
    late positions + 1 (a subset, and one doc at + 3), so a phrase (0, 1) has only late candidates.  Positions of term 1
    come first in the file, then pad bytes, then term 0, so that term 0's block data starts 4-byte aligned in memory.
    Returns a dict: pos (u8 file), po / pl (ranges), deltas (u32 view of the huge region), late (the late postings'
    deltas), index (the oracle index of the late postings of term 0 and all of term 1), docs / tfs per term, ids, total,
    data_off (byte offset of term 0's block data in the file), late_off (position offset of the first late posting)."""
    import phrase_oracle as O
    rng = np.random.default_rng(seed)
    late_pos = []
    for tf in late_tfs:
        d = rng.integers(1, 40, tf, dtype=np.int64)
        if tf > 50:
            d[tf // 2] = (1 << 31) + int(rng.integers(0, 1 << 20))   # late positions at and above 2^31
        late_pos.append(np.cumsum(d).astype(np.uint32))
    late = np.concatenate([np.diff(p, prepend=np.uint32(0)).astype(np.uint32) for p in late_pos])
    hb = n_huge * HUGE_TF // 128
    lb = late.size // 128
    late_blocks = [O._bitpack4x(late[b * 128:(b + 1) * 128]) for b in range(lb)]
    head = bytes(O._vint(hb + lb)) + bytes([32]) * hb + bytes(w for w, _ in late_blocks)
    tail = b"".join(p for _, p in late_blocks) + b"".join(bytes(O._vint(int(x))) for x in late[lb * 128:])
    # term 1: the partner's positions, serialized by the oracle writer
    ldocs = np.arange(n_huge, n_huge + len(late_tfs), dtype=np.uint32)
    p1, d1 = [], []
    for i, p in enumerate(late_pos):
        if i == 1:
            continue                                              # a late doc without the partner
        x = p[np.sort(rng.choice(p.size, max(1, p.size // 2), replace=False))].astype(np.int64)
        p1.append((x + (3 if i == 3 else 1)).astype(np.uint32)); d1.append(ldocs[i])
    t1 = O.serialize_positions(np.concatenate([np.diff(p, prepend=np.uint32(0)) for p in p1]).astype(np.uint32))
    pad = (-(len(t1) + len(head))) % 4
    data_off = len(t1) + pad + len(head)
    nbytes = data_off + hb * 512 + len(tail)
    pos = np.zeros(nbytes, np.uint8)
    pos[:len(t1)] = np.frombuffer(t1, np.uint8)
    pos[len(t1) + pad:data_off] = np.frombuffer(head, np.uint8)
    deltas = pos[data_off:data_off + hb * 512].view(np.uint32)
    step = 1 << 24
    for a in range(0, deltas.size, step):
        deltas[a:a + step] = rng.integers(0, 8, min(step, deltas.size - a), dtype=np.uint32)
    blk = deltas.reshape(hb, 128)
    blk[np.arange(hb), rng.integers(0, 128, hb)] = rng.integers(1 << 31, 1 << 32, hb, dtype=np.uint64).astype(np.uint32)
    pos[data_off + hb * 512:] = np.frombuffer(tail, np.uint8)
    po = np.array([len(t1) + pad, 0], np.uint64)
    pl = np.array([nbytes - len(t1) - pad, len(t1)], np.uint64)
    docs = [np.concatenate([np.arange(n_huge, dtype=np.uint32), ldocs]), np.array(d1, np.uint32)]
    tfs = [np.array([HUGE_TF] * n_huge + list(late_tfs), np.uint32), np.array([p.size for p in p1], np.uint32)]
    ids = rng.integers(0, 256, max_doc).astype(np.uint8)
    from stract_b200.bm25 import fieldnorm_table
    total = int(fieldnorm_table()[ids].astype(np.uint64).sum())
    index = {"fieldnorm_ids": ids, "total_num_tokens": total,
             "terms": [{"docs": ldocs, "positions": late_pos}, {"docs": docs[1], "positions": p1}]}
    late_off = n_huge * HUGE_TF
    # self-check: the late blocks start past 4 GiB of the term's data, the bytes parse back, a phrase matches there
    assert data_off % 4 == 0 and late_off * 4 > 1 << 32 and lb >= 2
    assert O.serialize_positions(late) == bytes(O._vint(lb)) + head[-lb:] + tail, "the late part as the writer has it"
    return {"pos": pos, "po": po, "pl": pl, "deltas": deltas, "late": late, "index": index, "docs": docs, "tfs": tfs, "ids": ids,
            "total": total, "data_off": data_off, "late_off": late_off, "n_huge": n_huge}
