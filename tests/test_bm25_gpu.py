"""Parity of the CUDA BM25 top-k path (through the C ABI) against the CPU oracle.  Needs a GPU.
Bar: doc ids, order and f32 scores / f64 totals bit-exact."""
import numpy as np
import pytest

import oracle
from stract_b200 import bm25
from stract_b200.bm25 import MODE_AND, MODE_OR, NO_TERM, SegmentReader, SignalComputer, SignalTable, TopDocs

pytestmark = pytest.mark.gpu


def total_num_tokens(ids):
    """The sum of the fieldnorms of `ids` (u8 fieldnorm codes) without a per-doc wide temporary: np.bincount casts its
    input to intp, so it runs over chunks (a 2^31-doc segment would otherwise take 17 GB)."""
    counts = np.zeros(256, np.uint64)
    for a in range(0, ids.size, 1 << 24):
        counts += np.bincount(ids[a:a + (1 << 24)], minlength=256).astype(np.uint64)
    return int((counts * bm25.fieldnorm_table().astype(np.uint64)).sum())


def build(term_docs, term_tfs, lens, record_option=1, fieldnorm_ids=None):
    """The same index as an oracle Segment and as a device SegmentReader (library writer).  `fieldnorm_ids` (u8 codes)
    replaces `lens` when given."""
    ids = bm25.fieldnorms_to_ids(lens) if fieldnorm_ids is None else np.ascontiguousarray(fieldnorm_ids, np.uint8)
    oseg = oracle.Segment(ids, record_option=record_option)
    for d, t in zip(term_docs, term_tfs):
        oseg.add_term(np.asarray(d, np.uint32), np.asarray(t, np.uint32))
    data, infos = bm25.encode_postings(term_docs, term_tfs, ids, oseg.avg_fieldnorm, record_option=record_option)
    assert np.array_equal(data, oseg.postings_bytes())
    seg = SegmentReader(data, infos, ids, record_option=record_option, total_num_tokens=total_num_tokens(ids))
    assert seg.average_fieldnorm == np.float32(oseg.avg_fieldnorm)
    return oseg, seg


def random_index(seed, max_doc, dfs, record_option=1):
    rng = np.random.default_rng(seed)
    lens = np.maximum(1, rng.lognormal(4.0, 0.8, max_doc)).astype(np.uint32)
    td, tt = [], []
    for df in dfs:
        td.append(np.sort(rng.choice(max_doc, df, replace=False)).astype(np.uint32))
        tt.append(np.minimum(rng.geometric(0.6, df), 255).astype(np.uint32))
    return build(td, tt, lens, record_option), rng


def weights_for(seg, q):
    w = np.array([bm25.Bm25Weight.for_one_term(int(seg.doc_freq[t]), seg.max_doc, seg.average_fieldnorm).weight for t in q], np.float32)
    cache = bm25.compute_tf_cache(seg.average_fieldnorm)
    return w, np.tile(cache, (len(q), 1))


def check_query(oseg, seg, q, mode, k, omode=None):
    w, caches = weights_for(seg, q)
    od, os_, _ = oseg.topk(np.array(q, np.uint32), w, caches, mode if omode is None else omode, k)
    got = TopDocs.with_limit(k).search(seg, q, mode)
    gd = np.array([d for _, d in got], np.uint32); gs = np.array([s for s, _ in got], np.float32)
    assert np.array_equal(gd, od), (q, mode, k, gd[:10], od[:10])
    assert np.array_equal(gs, os_), (q, mode, k)


def test_droopy_tax_kat():
    # tantivy/src/collector/top_score_collector.rs:590-602,676-700
    docs = ["hello happy tax payer".split(), "droopy says hello happy tax payer".split(), "i like droopy".split()]
    vocab = sorted({w for t in docs for w in t})
    td = [[d for d, t in enumerate(docs) if w in t] for w in vocab]
    tt = [[docs[d].count(w) for d in ds] for w, ds in zip(vocab, td)]
    oseg, seg = build(td, tt, [len(t) for t in docs])
    q = [vocab.index("droopy"), vocab.index("tax")]
    r = TopDocs.with_limit(4).search(seg, q, MODE_OR)
    assert [d for _, d in r] == [1, 2, 0]
    for (s, _), e in zip(r, (0.81221175, 0.5376842, 0.48527452)):
        assert abs(s - e) < 1e-6
    assert [d for _, d in TopDocs.with_limit(2).search(seg, q, MODE_OR)] == [1, 2]
    r = TopDocs.with_limit(4).search(seg, q, MODE_AND)
    assert [d for _, d in r] == [1] and abs(r[0][0] - 0.81221175) < 1e-6
    # and_offset, top_score_collector.rs:701-751
    r = TopDocs.with_limit(4).and_offset(2).search(seg, q, MODE_OR)
    assert [d for _, d in r] == [0] and abs(r[0][0] - 0.48527452) < 1e-6
    r = TopDocs.with_limit(2).and_offset(1).search(seg, q, MODE_OR)
    assert [d for _, d in r] == [2, 0] and abs(r[0][0] - 0.5376842) < 1e-6 and abs(r[1][0] - 0.48527452) < 1e-6


DFS = [1, 3, 100, 127, 128, 129, 255, 256, 257, 300, 511, 512, 1000, 1024, 2500, 6000, 15000, 40000]


def test_and_queries_bit_exact():
    (oseg, seg), rng = random_index(11, 60_000, DFS)
    nt = len(DFS)
    for _ in range(40):
        n = int(rng.integers(1, 5))
        q = [int(x) for x in rng.choice(nt, n, replace=False)]
        for k in (1, 10, 1000):
            check_query(oseg, seg, q, MODE_AND, k)
    # the two most frequent terms: thousands of matches -> exercises the buffer truncation
    check_query(oseg, seg, [nt - 1, nt - 2], MODE_AND, 100)
    check_query(oseg, seg, [nt - 1, nt - 2, nt - 3], MODE_AND, 1000)
    # a single clause above 65 536 postings sends its whole batch to k_topk_warp<AND>, the two-clause queries in it too
    (oseg, seg), _ = random_index(17, 100_000, [70_000, 500])
    for q in ([0], [0, 1]):
        for k in (10, 1000):
            check_query(oseg, seg, q, MODE_AND, k)
    terms = np.array([[0, NO_TERM], [0, 1], [1, 0]], np.uint32)
    gd, gs, gn = TopDocs.with_limit(1000).search_batch(seg, terms, MODE_AND)
    for q in range(len(terms)):
        qq = np.array([x for x in terms[q] if x != NO_TERM], np.uint32)
        od, os_, _ = oseg.topk(qq, *weights_for(seg, qq), MODE_AND, 1000)
        assert gn[q] == len(od), q
        assert np.array_equal(gd[q, :gn[q]], od) and np.array_equal(gs[q, :gn[q]], os_), q


def test_or_queries_bit_exact_up_to_two_terms():
    (oseg, seg), rng = random_index(12, 60_000, DFS)
    nt = len(DFS)
    for _ in range(30):
        n = int(rng.integers(1, 3))
        q = [int(x) for x in rng.choice(nt, n, replace=False)]
        for k in (1, 10, 1000):
            check_query(oseg, seg, q, MODE_OR, k)           # vs the reference's block_wand
            check_query(oseg, seg, q, MODE_OR, k, omode=2)  # vs the exhaustive union


def test_or_three_plus_terms_canonical_order():
    # documented deviation: the reference's f32 sum order for >= 3 OR terms depends on the pruning history;
    # the library sums in query order.  Bit-exact against the oracle's exhaustive union, and the doc SET /
    # scores agree with block_wand within 1 ulp-scale tolerance.
    (oseg, seg), rng = random_index(13, 60_000, DFS)
    nt = len(DFS)
    for _ in range(20):
        n = int(rng.integers(3, 6))
        q = [int(x) for x in rng.choice(nt, n, replace=False)]
        check_query(oseg, seg, q, MODE_OR, 200, omode=2)
        w, caches = weights_for(seg, q)
        bd, bs, _ = oseg.topk(np.array(q, np.uint32), w, caches, 1, 200)
        got = TopDocs.with_limit(200).search(seg, q, MODE_OR)
        gs = np.array([s for s, _ in got], np.float32)
        assert np.allclose(gs, bs, rtol=1e-6, atol=0)


def test_ties_order_by_doc_and_padding():
    n = 3000
    td = [np.arange(n, dtype=np.uint32), np.arange(0, n, 2, dtype=np.uint32)]
    tt = [np.ones(n, np.uint32), np.ones(n // 2, np.uint32)]
    oseg, seg = build(td, tt, [7] * n)
    r = TopDocs.with_limit(300).search(seg, [0], MODE_OR)
    assert [d for _, d in r] == list(range(300)) and len({s for s, _ in r}) == 1
    r = TopDocs.with_limit(50).search(seg, [0, 1], MODE_AND)
    assert [d for _, d in r] == list(range(0, 100, 2))
    # padding with NO_TERM == shorter query
    d1, s1, n1 = TopDocs.with_limit(50).search_batch(seg, np.array([[1, NO_TERM], [0, 1]], np.uint32), MODE_AND)
    assert n1[0] == 50 and list(d1[0]) == list(range(0, 100, 2)) and list(d1[1]) == list(range(0, 100, 2))
    # empty intersection
    oseg2, seg2 = build([np.array([1, 5, 9], np.uint32), np.array([2, 6, 10], np.uint32)], [np.ones(3, np.uint32)] * 2, [4] * 12)
    assert TopDocs.with_limit(10).search(seg2, [0, 1], MODE_AND) == []
    assert [d for _, d in TopDocs.with_limit(10).search(seg2, [0, 1], MODE_OR)] == [1, 2, 5, 6, 9, 10]


def test_batch_matches_oracle_batch():
    (oseg, seg), rng = random_index(14, 200_000, [int(x) for x in np.geomspace(200, 60000, 60)])
    nq = 400
    terms = np.stack([rng.choice(60, 2, replace=False) for _ in range(nq)]).astype(np.uint32)
    cache = bm25.compute_tf_cache(seg.average_fieldnorm)
    w = np.zeros((nq, 2), np.float32)
    for q in range(nq):
        for t in range(2):
            w[q, t] = bm25.Bm25Weight.for_one_term(int(seg.doc_freq[terms[q, t]]), seg.max_doc, seg.average_fieldnorm).weight
    caches = np.tile(cache, (nq * 2, 1))
    for mode in (MODE_AND, MODE_OR):
        od, os_, on, _ = oseg.topk_batch(terms, w, caches, mode, 1000, threads=8)
        gd, gs, gn, st = TopDocs.with_limit(1000).search_batch(seg, terms, mode, return_stats=True)
        assert np.array_equal(gn, on)
        for q in range(nq):
            assert np.array_equal(gd[q, :gn[q]], od[q, :on[q]]) and np.array_equal(gs[q, :gn[q]], os_[q, :on[q]])
        assert st["postings_scored"] == int(seg.doc_freq[terms].sum())


def test_signal_combine_bit_exact():
    (oseg, seg), rng = random_index(15, 80_000, [int(x) for x in np.geomspace(100, 30000, 40)])
    cols = [rng.random(80_000) ** 8, np.array([bm25.score_rank(r) for r in rng.permutation(80_000)]), rng.random(80_000),
            1.0 / (1.0 + rng.integers(0, 1000, 80_000))]
    coeffs = [2.0, 0.02, 2.0, 0.001]
    table = SignalTable(cols)
    comp = SignalComputer(seg, table, coeffs, coeff_text=0.005)
    nq = 60
    terms = np.stack([rng.choice(40, 5, replace=False) for _ in range(nq)]).astype(np.uint32)
    cache = bm25.compute_tf_cache(seg.average_fieldnorm)
    w = np.zeros((nq, 5), np.float32)
    for q in range(nq):
        for t in range(5):
            w[q, t] = bm25.StractBm25Weight.for_one_term(int(seg.doc_freq[terms[q, t]]), seg.max_doc, seg.average_fieldnorm).weight
    caches = np.tile(cache, (nq * 5, 1))
    for max_docs in (0, 5000, 137):
        od, ot, on, osc = oseg.signal_topk_batch(terms, w, caches, 1.2, 0.005, cols, coeffs, 100, max_docs=max_docs, threads=8)
        gd, gt, gn, st = comp.top_docs_batch(terms, 100, max_docs=max_docs, return_stats=True)
        assert np.array_equal(gn, on)
        for q in range(nq):
            assert np.array_equal(gd[q, :gn[q]], od[q, :on[q]]), (q, max_docs)
            assert np.array_equal(gt[q, :gn[q]], ot[q, :on[q]]), (q, max_docs)
        assert st["docs_scored"] == int(osc.sum())
    # no numeric signals: pure Stract BM25 ordering
    comp0 = SignalComputer(seg, None, (), coeff_text=1.0)
    od, ot, on, _ = oseg.signal_topk_batch(terms[:10], w[:10], caches[:50], 1.2, 1.0, [], [], 50)
    gd, gt, gn = comp0.top_docs_batch(terms[:10], 50)
    assert np.array_equal(gd, od) and np.array_equal(gt, ot)


def test_malformed_postings_rejected():
    from stract_b200._lib import Sb200Error
    (oseg, seg), rng = random_index(16, 5000, [300, 10])
    data = oseg.postings_bytes().copy()
    off, ln, df = oseg.term_infos()
    with pytest.raises(Sb200Error):
        SegmentReader(data, (off, ln, np.array([700, 10], np.uint32)), oseg.fieldnorm_ids)  # df disagrees with the skip list
    with pytest.raises(Sb200Error):
        SegmentReader(data[:100], (off, ln, df), oseg.fieldnorm_ids)  # term range outside the file


def test_and3_unit_kernel_bit_exact(monkeypatch):
    """The unit-based intersection (bm25_and3.cuh) against the oracle: ragged clause sizes (tail-only terms, exact
    multiples of 128), 1..4 clauses, k below/above the hit count, and a budget small enough to force several
    candidate groups."""
    dfs = [1, 5, 127, 128, 129, 255, 256, 300, 1000, 1280, 5000, 20000, 40000]
    (oseg, seg), rng = random_index(21, 80_000, dfs)
    nt = len(dfs)
    for _ in range(60):
        n = int(rng.integers(1, 5))
        q = [int(x) for x in rng.choice(nt, n, replace=False)]
        for k in (1, 10, 1000):
            check_query(oseg, seg, q, MODE_AND, k)
    check_query(oseg, seg, [nt - 1, nt - 2], MODE_AND, 100)
    check_query(oseg, seg, [nt - 1], MODE_AND, 4096)          # single clause: every posting is a hit, chunked select
    check_query(oseg, seg, [nt - 1, nt - 2, nt - 3], MODE_AND, 1000)
    # batch + forced grouping of the candidate memory
    monkeypatch.setenv("SB200_AND3_BUDGET_MB", "1")
    nq = 300
    terms = np.stack([rng.choice(nt, 2, replace=False) for _ in range(nq)]).astype(np.uint32)
    cache = bm25.compute_tf_cache(seg.average_fieldnorm)
    w = np.zeros((nq, 2), np.float32)
    for q in range(nq):
        for t in range(2):
            w[q, t] = bm25.Bm25Weight.for_one_term(int(seg.doc_freq[terms[q, t]]), seg.max_doc, seg.average_fieldnorm).weight
    caches = np.tile(cache, (nq * 2, 1))
    od, os_, on, _ = oseg.topk_batch(terms, w, caches, MODE_AND, 1000, threads=8)
    gd, gs, gn, st = TopDocs.with_limit(1000).search_batch(seg, terms, MODE_AND, return_stats=True)
    assert np.array_equal(gn, on)
    for q in range(nq):
        assert np.array_equal(gd[q, :gn[q]], od[q, :on[q]]) and np.array_equal(gs[q, :gn[q]], os_[q, :on[q]])
    assert st["docs_scored"] == int(on.sum()) or st["docs_scored"] >= int(on.sum())


def union_kernel_against_oracle(seed, max_doc, dfs, nq, ks, pad_every, sig_nq, sig_k):
    """k_or3 against the oracle on a random index (see union_kernel_check)."""
    (oseg, seg), rng = random_index(seed, max_doc, dfs)
    union_kernel_check(oseg, seg, rng, nq, ks, pad_every, sig_nq, sig_k)


def union_kernel_check(oseg, seg, rng, nq, ks, pad_every, sig_nq, sig_k, sig_cols=(4, 2, 0), sig_max_docs=(0,)):
    """k_or3 against the oracle: OR batches of 1/2/3/5/8 clauses (every `pad_every`-th query of 3+ clauses padded with
    NO_TERM) whose large queries are cut into doc-range items and merged, compared query by query with the exhaustive
    union; and the signal combine with `sig_cols` columns (k_or3, or k_topk_warp for a max_docs cut)."""
    nt, max_doc = seg.n_terms, seg.max_doc
    for width in (1, 2, 3, 5, 8):
        terms = np.stack([rng.choice(nt, width, replace=False) for _ in range(nq)]).astype(np.uint32)
        if width >= 3:
            terms[::pad_every, 1] = NO_TERM   # padded / absent clauses
        for k in ks:
            gd, gs, gn = TopDocs.with_limit(k).search_batch(seg, terms, MODE_OR)
            for q in range(nq):
                qq = np.array([x for x in terms[q] if x != NO_TERM], np.uint32)
                w, caches = weights_for(seg, qq)
                od, os_, _ = oseg.topk(qq, w, caches, 2, k)      # oracle mode 2 = exhaustive union
                m = int(gn[q])
                assert m == len(od), (width, k, q, m, len(od))
                assert np.array_equal(gd[q, :m], od) and np.array_equal(gs[q, :m], os_), (width, k, q)
    cache = bm25.compute_tf_cache(seg.average_fieldnorm)
    for ncols in sig_cols:
        cols = [rng.random(max_doc) for _ in range(ncols)]
        coeffs = [2.0, 0.02, 2.0, 0.001][:ncols]
        comp = SignalComputer(seg, SignalTable(cols) if ncols else None, coeffs, coeff_text=0.005)
        terms = np.stack([rng.choice(nt, 5, replace=False) for _ in range(sig_nq)]).astype(np.uint32)
        w = np.array([[bm25.StractBm25Weight.for_one_term(int(seg.doc_freq[t]), seg.max_doc, seg.average_fieldnorm).weight for t in row]
                      for row in terms], np.float32)
        for max_docs in sig_max_docs:
            od, ot, on, _ = oseg.signal_topk_batch(terms, w, np.tile(cache, (sig_nq * 5, 1)), 1.2, 0.005, cols, coeffs, sig_k,
                                                   max_docs=max_docs, threads=8)
            gd, gt, gn = comp.top_docs_batch(terms, sig_k, max_docs=max_docs)
            assert np.array_equal(gn, on), (ncols, max_docs)
            for q in range(sig_nq):
                assert np.array_equal(gd[q, :gn[q]], od[q, :on[q]]) and np.array_equal(gt[q, :gn[q]], ot[q, :on[q]]), (ncols, max_docs, q)


def test_or3_union_kernel_bit_exact():
    union_kernel_against_oracle(31, 200_000, [1, 5, 127, 128, 129, 300, 1000, 1280, 5000, 20000, 40000, 60000, 90000],
                                nq=120, ks=(1, 10, 1000), pad_every=7, sig_nq=80, sig_k=1000)


def test_or_wand_replay_matches_block_wand_bit_for_bit():
    """SB200_MODE_OR_WAND: tantivy's block_wand replayed on the device -- docs, order and f32 score bits equal the oracle's
    block_wand (mode 1) for 1..8 terms, small and large k, tie-heavy data (few distinct lengths / tfs)."""
    from stract_b200.bm25 import MODE_OR_WAND
    rng = np.random.default_rng(77)
    max_doc = 50_000
    lens = rng.choice([3, 5, 8, 13, 40], max_doc).astype(np.uint32)          # few fieldnorms: many exactly tied term scores
    dfs = [1, 40, 127, 128, 129, 500, 2000, 2600, 9000, 20000, 30000]
    td, tt = [], []
    for df in dfs:
        td.append(np.sort(rng.choice(max_doc, df, replace=False)).astype(np.uint32))
        tt.append(rng.choice([1, 1, 1, 2, 3], df).astype(np.uint32))
    oseg, seg = build(td, tt, lens)
    flips = 0
    for width, k in ((1, 10), (2, 25), (3, 10), (3, 300), (5, 10), (5, 1000), (8, 100)):
        nq = 12
        terms = np.stack([rng.choice(len(dfs), width, replace=False) for _ in range(nq)]).astype(np.uint32)
        d, s, n = TopDocs.with_limit(k).search_batch(seg, terms, MODE_OR_WAND)
        dx, sx, nx = TopDocs.with_limit(k).search_batch(seg, terms, MODE_OR)
        for q in range(nq):
            w, caches = weights_for(seg, terms[q])
            od, os_, _ = oseg.topk(terms[q], w, caches, 1, k)      # oracle mode 1 = block_wand
            m = int(n[q])
            assert m == len(od), (width, k, q, m, len(od))
            assert np.array_equal(d[q, :m], od), (width, k, q)
            assert np.array_equal(s[q, :m], os_), (width, k, q)
            flips += int(not np.array_equal(s[q, :m], sx[q, :m]))
    # absent clauses are dropped like in the other modes
    t = np.array([[10, NO_TERM, 9, 8], [NO_TERM, 7, 6, 5]], np.uint32)
    d, s, n = TopDocs.with_limit(50).search_batch(seg, t, MODE_OR_WAND)
    for q in range(2):
        qq = [int(x) for x in t[q] if x != NO_TERM]
        w, caches = weights_for(seg, qq)
        od, os_, _ = oseg.topk(np.array(qq, np.uint32), w, caches, 1, 50)
        assert np.array_equal(d[q, :n[q]], od) and np.array_equal(s[q, :n[q]], os_)
    print("queries whose score bits differ between the replay and the query-order union:", flips)


def test_packed_result_copy_equals_dense(monkeypatch):
    """Sparse AND tables leave the device packed (copy_out_tables); same docs / scores / counts as the dense copy."""
    dfs = [1, 5, 127, 128, 129, 300, 1000, 1280, 5000, 12000]
    (oseg, seg), rng = random_index(91, 60_000, dfs)
    terms = np.stack([rng.choice(len(dfs), 2, replace=False) for _ in range(64)]).astype(np.uint32)
    monkeypatch.setenv("SB200_BM25_DENSE_OUT", "1")
    d0, s0, n0 = TopDocs.with_limit(500).search_batch(seg, terms, MODE_AND)
    d0, s0, n0 = d0.copy(), s0.copy(), n0.copy()
    monkeypatch.delenv("SB200_BM25_DENSE_OUT")
    monkeypatch.setenv("SB200_BM25_PACK_MIN", "1")
    d1, s1, n1 = TopDocs.with_limit(500).search_batch(seg, terms, MODE_AND)
    assert np.array_equal(n0, n1) and int(n1.sum()) * 2 < terms.shape[0] * 500
    for q in range(terms.shape[0]):
        assert np.array_equal(d0[q, :n0[q]], d1[q, :n1[q]]) and np.array_equal(s0[q, :n0[q]], s1[q, :n1[q]])
