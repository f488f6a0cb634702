"""Phrase queries on the device (sb200_phrase_topk_batch) bit-exact against the CPU oracle (tests/phrase_oracle.py): docs,
order and f32 score bits."""
import numpy as np
import pytest

import phrase_oracle as O
from phrase_fixtures import assert_same, make_segment, oracle_batch, random_index, random_rows

pytestmark = pytest.mark.gpu


def check_random_batches(n_docs=6000, nq=24, widths=(2, 3, 5, 8), seed=11):
    from stract_b200.bm25 import TopDocs
    index, rng = random_index(seed, n_docs)
    seg = make_segment(index)
    nv = len(index["terms"]) - 2
    for width in widths:
        rows, offs = random_rows(rng, nv, nq, width)
        for slop in (0, 1, 2, 3, 300):
            slops = np.full(nq, slop, np.uint32)
            for scoring in (True, False):
                for k in ((1, 10, 1000) if slop in (0, 2) else (1000,)):
                    got = TopDocs.with_limit(k).search_phrase_batch(seg, rows, offs, slops, scoring)
                    assert_same(got, oracle_batch(index, rows, offs, slops, scoring, k))
    # the long document's tf (1500 per term) is above the shared buffer
    from stract_b200.bm25 import NO_TERM
    rows = np.array([[0, 1, NO_TERM], [1, 0, 1], [0, 1, 0]], np.uint32)
    offs = np.array([[0, 1, 0], [0, 1, 2], [0, 1, 2]], np.uint32)
    for slop in (0, 1, 3):
        for scoring in (True, False):
            slops = np.full(3, slop, np.uint32)
            got = TopDocs.with_limit(4096).search_phrase_batch(seg, rows, offs, slops, scoring, return_stats=True)
            assert_same(got[:3], oracle_batch(index, rows, offs, slops, scoring, 4096))
            assert 0 in set(got[0][0, :got[2][0]].tolist())
    seg.close()


def test_phrases_bit_exact_against_oracle():
    check_random_batches()


def check_reference_phrase_tests():
    """The reference's phrase_query/mod.rs tests through the library (scores within assert_nearly_equals and bit-equal to
    the oracle)."""
    from stract_b200.bm25 import PhraseQuery, TopDocs
    cases = [(["a b c", "a b c a b"], ["a", "b"], 0, [0.40618482, 0.46844664]),
             (["a b e c", "a e e e c", "a e e e e c"], ["a", "c"], 3, [0.29086056, 0.26706287]),
             (["a e b e c", "a e e e e e b e e e e c", "a c b", "a c e b e", "a e c b", "a e b c"], ["a", "b", "c"], 3,
              {0: 0.23091172, 1: 0.27310878, 3: 0.25024384})]
    for texts, query, slop, want in cases:
        index, vocab = O.build_index(texts)
        seg = make_segment(index)
        q = PhraseQuery([vocab[t] for t in query], slop=slop)
        rows, offs, slops = PhraseQuery.rows([q])
        d, s, n = TopDocs.with_limit(100).search_phrase_batch(seg, rows, offs, slops)
        by_doc = sorted(zip(d[0, :n[0]].tolist(), s[0, :n[0]].tolist()))
        want = dict(enumerate(want)) if isinstance(want, list) else want
        for i, v in want.items():
            assert abs(by_doc[i][1] - v) * 2 / (by_doc[i][1] + v) < 5e-4
        assert_same((d, s, n), oracle_batch(index, rows, offs, slops, True, 100))
        seg.close()
    index, vocab = O.build_index(["b", "a b", "b a"])
    seg = make_segment(index)
    rows, offs, slops = PhraseQuery.rows([PhraseQuery([vocab["a"], vocab["b"]]), PhraseQuery([vocab["b"], vocab["a"]])])
    d, s, n = TopDocs.with_limit(10).search_phrase_batch(seg, rows, offs, slops)
    assert list(n) == [1, 1] and d[0, 0] == 1 and d[1, 0] == 2
    seg.close()
    index, vocab = O.build_index(["b c x x a b", "c b a"])   # phrase_exists vs count > 0 (test_oracle_phrase)
    seg = make_segment(index)
    rows, offs, slops = PhraseQuery.rows([PhraseQuery([vocab[t] for t in "cba"], slop=2)])
    for scoring, docs in ((True, [1]), (False, [0, 1])):
        d, s, n = TopDocs.with_limit(10).search_phrase_batch(seg, rows, offs, slops, scoring)
        assert d[0, :n[0]].tolist() == docs
    seg.close()


def test_reference_phrase_tests():
    check_reference_phrase_tests()


def check_positions_read_kats():
    """positions/mod.rs reader KATs through sb200_positions_read (one term per KAT stream)."""
    from stract_b200.bm25 import SegmentReader, encode_positions, encode_postings
    streams = [np.arange(1000), np.arange(512), np.arange(2_000_000), np.full(2_000_000, 9)]
    # one posting per term whose absolute positions are the running sum of the KAT deltas
    absolute = [np.cumsum(s.astype(np.uint64)).astype(np.uint32) for s in streams]
    tfs = np.array([s.size for s in streams], np.uint32)
    pos, po, pl = encode_positions(np.concatenate(absolute), tfs, np.arange(5))
    assert list(pl) == [1224, 533, 5_003_499, 1_015_627]
    ids = np.ones(1, np.uint8)
    data, infos = encode_postings([[0]] * 4, [[int(t)] for t in tfs], ids, 1.0, record_option=2)
    seg = SegmentReader(data, infos, ids, record_option=2, total_num_tokens=1, positions=pos, positions_ranges=(po, pl))
    for n in (1, 10, 127, 128, 130, 312):
        assert np.array_equal(seg.read_positions(0, 0, n), np.arange(n))
    for off in (1, 10, 127, 128, 130, 312):
        for ln in (1, 10, 130, 500):
            assert np.array_equal(seg.read_positions(0, off, ln), np.arange(off, off + ln))
    for off in range(0, 700, 7):
        assert np.array_equal(seg.read_positions(0, off, 7), np.arange(off, off + 7))
    assert seg.read_positions(1, 230, 1)[0] == 230 and seg.read_positions(1, 9, 1)[0] == 9
    assert np.array_equal(seg.read_positions(2, 128, 256), np.arange(128, 384))
    for off in (10, 128 * 1024, 128 * 1024 - 1, 128 * 1024 + 7, 128 * 10 * 1024 + 10):
        assert seg.read_positions(2, off, 1)[0] == off
    assert seg.read_positions(3, 0, 1)[0] == 9
    from stract_b200._lib import Sb200Error
    with pytest.raises(Sb200Error):
        seg.read_positions(0, 999, 2)
    info = seg.info()
    seg.close()
    return info


def test_positions_read_kats():
    check_positions_read_kats()


def check_error_paths():
    from stract_b200._lib import Sb200Error
    from stract_b200.bm25 import SegmentReader, TopDocs, encode_postings
    index, vocab = O.build_index(["a b c", "a b"])
    seg = make_segment(index)
    rows = np.array([[vocab["a"], vocab["b"]]], np.uint32)
    with pytest.raises(Sb200Error):   # a one-term phrase
        TopDocs.with_limit(5).search_phrase_batch(seg, np.array([[vocab["a"], 0xFFFFFFFF]], np.uint32))
    bad_pos = np.array([5], np.uint8)
    with pytest.raises(Sb200Error):   # ranges outside the file
        seg.attach_positions(bad_pos, (np.array([0, 0, 9], np.uint64), np.array([1, 1, 1], np.uint64)))
    with pytest.raises(Sb200Error):   # an unterminated VInt header
        seg.attach_positions(np.array([5, 5, 5], np.uint8), (np.array([0, 1, 2], np.uint64), np.array([1, 1, 1], np.uint64)))
    with pytest.raises(Sb200Error):   # the failed attach left the segment without positions
        TopDocs.with_limit(5).search_phrase_batch(seg, rows)
    seg.close()
    ids = index["fieldnorm_ids"]
    tfs = [np.array([len(p) for p in t["positions"]], np.uint32) for t in index["terms"]]
    data, infos = encode_postings([t["docs"] for t in index["terms"]], tfs, ids, 2.5, record_option=1)
    s1 = SegmentReader(data, infos, ids, record_option=1, total_num_tokens=5)
    with pytest.raises(Sb200Error):   # record option 1: no positions (PhraseQuery's SchemaError)
        TopDocs.with_limit(5).search_phrase_batch(s1, rows)
    with pytest.raises(Sb200Error):
        s1.attach_positions(np.array([128], np.uint8), (np.zeros(3, np.uint64), np.ones(3, np.uint64)))
    s1.close()


def test_error_paths():
    check_error_paths()


def check_term_info_store_positions():
    import oracle
    from stract_b200 import bm25
    n = 1000   # ranges are contiguous in a TermInfoStore: a term's end is the next term's start
    edges = np.concatenate([[0], np.cumsum(np.arange(n, dtype=np.uint64) % 7 + 1)]).astype(np.uint64)
    qedges = np.concatenate([[5], 5 + np.cumsum(np.arange(n, dtype=np.uint64) % 11 * 3)]).astype(np.uint64)
    store = oracle.term_info_store_write(np.arange(n, dtype=np.uint32), edges[:-1], edges[1:], qedges[:-1], qedges[1:])
    po, pl = bm25.decode_term_info_store_positions(store)
    assert np.array_equal(po, qedges[:-1]) and np.array_equal(pl, np.diff(qedges))
    infos, cnt = bm25.decode_term_info_store(store)
    assert cnt == n and [infos[i].postings_off for i in range(n)] == edges[:-1].tolist()


def test_term_info_store_positions_range():
    check_term_info_store_positions()


def check_searcher_three_segments():
    from stract_b200.bm25 import ABSENT_TERM, Searcher, TopDocs
    index, rng = random_index(21, 3000, long_doc=50)
    n = index["fieldnorm_ids"].size
    cuts = [0, 1000, 2100, n]
    parts, ords = [], []
    for a, b in zip(cuts[:-1], cuts[1:]):
        terms, remap = [], {}
        for t, term in enumerate(index["terms"]):
            m = (term["docs"] >= a) & (term["docs"] < b)
            if m.any():
                remap[t] = len(terms)
                terms.append({"docs": term["docs"][m] - a, "positions": [p for p, k in zip(term["positions"], m) if k]})
        ids = index["fieldnorm_ids"][a:b]
        from stract_b200.bm25 import fieldnorm_table
        parts.append({"fieldnorm_ids": ids, "terms": terms, "total_num_tokens": int(fieldnorm_table()[ids].astype(np.uint64).sum())})
        ords.append(remap)
    segs = [make_segment(p) for p in parts]
    big = make_segment(index)
    rows, offs = random_rows(rng, len(index["terms"]) - 2, 16, 4, absent=False)
    per = [np.vectorize(lambda t, r=r: r.get(int(t), ABSENT_TERM) if t != 0xFFFFFFFF else 0xFFFFFFFF, otypes=[np.uint32])(rows) for r in ords]
    for slop in (0, 2):
        for scoring in (True, False):
            sl = np.full(16, slop, np.uint32)
            so, sd, ss, sn = Searcher(segs).search_phrase_batch(TopDocs.with_limit(50), per, offs, sl, scoring)
            bd, bs, bn = TopDocs.with_limit(50).search_phrase_batch(big, rows, offs, sl, scoring)
            assert np.array_equal(sn, bn)
            for q in range(16):
                glob = np.array([cuts[int(o)] for o in so[q, :sn[q]]], np.int64) + sd[q, :sn[q]]
                assert np.array_equal(glob, bd[q, :bn[q]]) and np.array_equal(ss[q, :sn[q]], bs[q, :bn[q]]), (slop, scoring, q)
    for s in segs + [big]:
        s.close()


def test_searcher_over_three_segments_matches_one_big_segment():
    check_searcher_three_segments()


def check_and_or_unchanged_by_positions():
    from stract_b200.bm25 import MODE_AND, MODE_OR, SegmentReader, TopDocs, encode_postings
    index, rng = random_index(5, 3000, long_doc=40)
    with_pos = make_segment(index)
    ids = index["fieldnorm_ids"]
    tfs = [np.array([len(p) for p in t["positions"]], np.uint32) for t in index["terms"]]
    avg = np.float32(np.float32(index["total_num_tokens"]) / np.float32(ids.size))
    data, infos = encode_postings([t["docs"] for t in index["terms"]], tfs, ids, avg, record_option=2)
    plain = SegmentReader(data, infos, ids, record_option=2, total_num_tokens=index["total_num_tokens"])
    rows = np.stack([rng.choice(len(index["terms"]), 3, replace=False) for _ in range(20)]).astype(np.uint32)
    for mode in (MODE_AND, MODE_OR):
        ad, as_, an = TopDocs.with_limit(100).search_batch(with_pos, rows, mode)
        bd, bs, bn = TopDocs.with_limit(100).search_batch(plain, rows, mode)
        assert np.array_equal(an, bn)
        for q in range(rows.shape[0]):
            assert np.array_equal(ad[q, :an[q]], bd[q, :bn[q]]) and np.array_equal(as_[q, :an[q]].view(np.uint32), bs[q, :bn[q]].view(np.uint32))
    assert with_pos.info()["hbm_bytes"] > plain.info()["hbm_bytes"]
    with_pos.close(); plain.close()


def test_and_or_results_unchanged_when_positions_attached():
    check_and_or_unchanged_by_positions()
