"""The phrase-query oracle (tests/phrase_oracle.py) pinned on the reference's own tests, and the library's positions writer
against it.  No GPU needed."""
import numpy as np
import pytest

import phrase_oracle as O


def _kat_bytes(deltas):
    return O.serialize_positions(deltas)


def test_positions_codec_sizes():
    # positions/mod.rs:90,137,155,178,196,211,223
    assert len(_kat_bytes(range(1000))) == 1224
    assert len(_kat_bytes(range(512))) == 533
    assert len(_kat_bytes(np.full(2_000_000, 9, np.uint32))) == 1_015_627


def test_positions_codec_size_two_million():
    assert len(_kat_bytes(range(2_000_000))) == 5_003_499


def test_position_reads():
    data = _kat_bytes(range(1000))
    for n in (1, 10, 127, 128, 130, 312):                       # test_position_read
        assert list(O.read_positions(data, 0, n)) == list(range(n))
    for off in (1, 10, 127, 128, 130, 312):                     # test_position_read_with_offset
        for ln in (1, 10, 130, 500):
            assert list(O.read_positions(data, off, ln)) == list(range(off, off + ln))
    for off in range(0, 700, 7):                                # test_position_read_after_skip (re-read at every step)
        assert list(O.read_positions(data, off, 7)) == list(range(off, off + 7))
    data = _kat_bytes(range(512))                               # test_position_requesting_passed_block
    assert O.read_positions(data, 230, 1)[0] == 230 and O.read_positions(data, 9, 1)[0] == 9
    data = _kat_bytes([1, 12, 4, 17, 443])                      # test_multiple_write_positions
    assert list(O.read_positions(data, 0, 5)) == [1, 12, 4, 17, 443]
    assert list(O.read_positions(_kat_bytes([]), 0, 0)) == []   # test_empty_position


def test_intersection_kats():
    # phrase_scorer.rs:575-582
    for l, r, e in [([1], [1], [1]), ([1], [2], []), ([], [2], []), ([5, 7], [1, 5, 10, 12], [5]),
                    ([1, 5, 6, 9, 10, 12], [6, 8, 9, 12], [6, 9, 12])]:
        for a, b in ((l, r), (r, l)):
            assert O.intersection_count(a, b) == len(e)
            assert O.intersection(a, b) == e
            assert O.intersection_exists(a, b) == bool(e)


@pytest.mark.parametrize("left,right,expected,slop", [
    ([1], [2], [2], 1), ([1], [3], [], 1), ([1], [3], [3], 2), ([], [2], [], 100000),
    ([5, 7, 11], [1, 5, 10, 12], [5, 10], 1), ([1, 5, 6, 9, 10, 12], [6, 8, 9, 12], [6, 8, 9, 12], 1),
    ([1, 5, 6, 9, 10, 12], [6, 8, 9, 12], [6, 8, 9, 12], 10), ([1, 3, 5], [2, 4, 6], [2, 4, 6], 1),
    ([1, 2], [1], [1], 1), ([3], [4], [4], 2)])    # test_slop + test_merge_slop, phrase_scorer.rs:583-611
def test_slop_and_merge_kats(left, right, expected, slop):
    c, out = O.intersection_count_with_slop(list(left), list(right), slop, True)
    assert out == expected and c == len(expected)
    assert O.intersection_exists_with_slop(left, right, slop) == bool(expected)


def test_slop_zero_kat():
    assert O.intersection([1, 3, 5], [2, 4, 6]) == []


@pytest.mark.parametrize("lists,expected,slop,count", [
    ([[1], []], [], 1, 0), ([[1], [2]], [(1, 1), (1, 2)], 1, 1), ([[1], [3]], [], 1, 0),
    ([[1], [2], [2]], [(1, 2)], 1, 1), ([[2], [1], [2]], [(1, 2)], 1, 1), ([[2], [2], [1]], [(1, 1), (1, 2)], 1, 1),
    ([[2], [2], [1], [2]], [(1, 2)], 1, 1), ([[1], [2], [2], [2]], [(1, 2)], 1, 1), ([[1], [2], [1]], [(1, 1)], 1, 1),
    ([[11], [10, 12]], [(1, 10), (1, 11), (1, 12)], 1, 1), ([[10, 12], [11]], [(1, 10), (1, 11), (1, 12)], 1, 1),
    ([[5, 7, 11], [1, 5, 10, 12]], [(0, 5), (1, 10), (1, 11), (1, 12)], 1, 2)])   # phrase_scorer.rs:642-668
def test_carrying_slop_kats(lists, expected, slop, count):
    left, slops = list(lists[0]), [0] * len(lists[0])
    c = 0
    for r in lists[1:]:
        c, left, slops = O.intersection_count_with_carrying_slop(left, slops, list(r), slop, True)
    assert list(zip(slops, left)) == expected and c == count


def _search(texts, query, slop=0, scoring=True, offsets=None):
    idx, vocab = O.build_index(texts)
    n = len(texts)
    terms = [vocab.get(t) for t in query]
    dfs = [0 if t is None else len(idx["terms"][t]["docs"]) for t in terms]
    avg = np.float32(np.float32(idx["total_num_tokens"]) / np.float32(n))
    w = O.bm25_weight_for_terms(dfs, n)
    cache = O.tf_cache(avg, np.arange(256))    # fieldnorm ids < 24 are the identity
    order = sorted(range(len(terms)), key=lambda i: (offsets or list(range(len(terms))))[i])
    t = [terms[i] for i in order]
    o = None if offsets is None else [offsets[i] for i in order]
    hits = O.phrase_search(idx, t, o, slop, scoring, w, cache)
    return sorted(hits, key=lambda h: h[1])    # the reference's test collectors list documents in doc order


def _docs(texts, query, **kw):
    return [d for _, d in _search(texts, query, **kw)]


def _scores(texts, query, **kw):
    return [float(s) for s, _ in _search(texts, query, **kw)]


def _near(a, b):   # assert_nearly_equals (tantivy/src/lib.rs): relative 5e-4
    return abs(a - b) * 2 / (abs(a) + abs(b)) < 5e-4


FIVE = ["b b b d c g c", "a b b d c g c", "a b a b c", "c a b a d ga a", "a b c"]


@pytest.mark.parametrize("scoring", [True, False])
def test_phrase_query_docsets(scoring):
    assert _docs(FIVE, ["a", "b"], scoring=scoring) == [1, 2, 3, 4]
    assert _docs(FIVE, ["a", "b", "c"], scoring=scoring) == [2, 4]
    assert _docs(FIVE, ["b", "b"], scoring=scoring) == [0, 1]
    assert _docs(FIVE, ["g", "ewrwer"], scoring=scoring) == []
    assert _docs(FIVE, ["g", "a"], scoring=scoring) == []
    assert _docs(["a b b d c g c", "a b a b c"], ["a", "b", "c"], scoring=False) == [1]   # test_phrase_query_simple


def test_phrase_scores():
    s = _scores(["a b c", "a b c a b"], ["a", "b"])
    assert _near(s[0], 0.40618482) and _near(s[1], 0.46844664)
    assert len(_scores(["asdf asdf Captain Subject Wendy", "Captain"], ["captain", "wendy"], slop=1)) == 1
    assert len(_scores(["a x b x c", "a a c"], ["a", "b", "c"], slop=2)) == 1
    assert len(_scores(["a x b x c", "b c c"], ["a", "b", "c"], slop=2)) == 1
    assert len(_scores(["wendy subject subject captain", "Captain"], ["wendy", "subject", "captain"], slop=1)) == 1
    s = _scores(["a b e c", "a e e e c", "a e e e e c"], ["a", "c"], slop=3)
    assert len(s) == 2 and _near(s[0], 0.29086056) and _near(s[1], 0.26706287)
    assert len(_scores(["a x b c"], ["a", "b", "c"], slop=1)) == 1
    assert len(_scores(["a x b x c"], ["a", "b", "c"], slop=1)) == 0
    assert len(_scores(["a b"], ["b", "a"], slop=1)) == 0
    assert len(_scores(["a b"], ["b", "a"], slop=2)) == 1
    s = _scores(["a e b e c", "a e e e e e b e e e e c", "a c b", "a c e b e", "a e c b", "a e b c"], ["a", "b", "c"], slop=3)
    assert _near(s[0], 0.23091172) and _near(s[1], 0.27310878) and _near(s[3], 0.25024384)


def test_phrase_docfreq_order_and_offsets():
    texts = ["b", "a b", "b a"]
    assert _docs(texts, ["a", "b"]) == [1]
    assert _docs(texts, ["b", "a"]) == [2]
    t = ["a b c d e f g h"]
    assert _docs(t, ["a", "b"], offsets=[0, 1]) == [0]
    assert _docs(t, ["b", "a"], offsets=[1, 0]) == [0]
    assert _docs(t, ["a", "b"], offsets=[0, 2]) == []
    assert _docs(t, ["a", "c"], offsets=[0, 2]) == [0]
    assert _docs(t, ["a", "c", "d"], offsets=[0, 2, 3]) == [0]
    assert _docs(t, ["a", "c", "e"], offsets=[0, 2, 4]) == [0]
    assert _docs(t, ["e", "a", "c"], offsets=[4, 0, 2]) == [0]
    assert _docs(t, ["a", "d"], offsets=[0, 2]) == []
    assert _docs(t, ["a", "c"], offsets=[1, 3]) == [0]


# With scoring off, phrase_exists ends with the NON-carrying intersection_exists_with_slop, so for >= 3 terms with slop the
# docset can differ from count > 0 (found by a search over short random documents)
DIFF_TEXTS, DIFF_QUERY, DIFF_SLOP = ["b c x x a b", "c b a"], ["c", "b", "a"], 2


def test_exists_differs_from_count_with_carrying_slop():
    assert _docs(DIFF_TEXTS, DIFF_QUERY, slop=DIFF_SLOP) == [1]
    assert _docs(DIFF_TEXTS, DIFF_QUERY, slop=DIFF_SLOP, scoring=False) == [0, 1]


def test_library_writer_equals_oracle_writer():
    from stract_b200.bm25 import encode_positions
    rng = np.random.default_rng(5)
    term_pos, tfs, offs = [], [], [0]
    idx = {"terms": []}
    for npost in (0, 1, 3, 40, 129, 300):
        plist = []
        for _ in range(npost):
            tf = int(rng.integers(1, 9)) if rng.random() < 0.9 else 300
            p = np.sort(rng.choice(5000, tf, replace=False)).astype(np.uint32)
            plist.append(p); term_pos.append(p); tfs.append(tf)
        idx["terms"].append({"positions": plist})
        offs.append(offs[-1] + npost)
    data, po, pl = encode_positions(np.concatenate(term_pos), np.array(tfs), np.array(offs))
    odata, opo, opl = O.positions_file(idx)
    assert np.array_equal(data, odata) and np.array_equal(po, opo) and np.array_equal(pl, opl)
    # the raw-delta KATs through the library writer: one posting whose absolute positions are the deltas' running sum
    for deltas in (np.arange(1000), np.arange(512), np.full(2_000_000, 9)):
        absolute = np.cumsum(deltas.astype(np.uint64)).astype(np.uint32)
        d, _, _ = encode_positions(absolute, [deltas.size], [0, 1])
        assert d.tobytes() == O.serialize_positions(deltas)


def test_carrying_slop_distance_wraps_in_u32():
    """`slop_so_far as u32 + abs_diff` wraps in the reference's release build (phrase_scorer.rs:270,317,327): a left
    position carrying slop 1 and a right position 2^32 - 1 away are at distance 0.  Hand-made lists for the main loop and
    both finish-rest branches, then a three-term phrase over one document, in the Python and the native oracle."""
    top = 0xFFFFFFFF
    c, left, slops = O.intersection_count_with_carrying_slop([0], [], [1], 1, True)
    assert (c, left, slops) == (1, [0, 1], [1, 1])
    assert O.intersection_count_with_carrying_slop(left, slops, [top], 1, False)[0] == 1        # main loop
    assert O.intersection_count_with_carrying_slop([0], [1], [5, top], 1, True) == (0, [top], [0])      # left exhausted
    assert O.intersection_count_with_carrying_slop([5, top], [1, 1], [0], 1, True) == (0, [top], [0])   # right exhausted
    assert O.intersection_count_with_carrying_slop([0], [1], [top - 1], 1, True) == (0, [], [])         # no wrap: 2^32 - 1
    from phrase_fixtures import index_to_csr, native_batch
    one = lambda p: {"docs": np.array([0], np.uint32), "positions": [np.array([p], np.uint32)]}
    idx = {"fieldnorm_ids": np.array([3], np.uint8), "terms": [one(0), one(1), one(top)], "total_num_tokens": 3}
    cache = O.tf_cache(np.float32(3.0), np.arange(256))
    w = O.bm25_weight_for_terms([1, 1, 1], 1)
    for slop, n in ((1, 1), (300, 1), (0, 0)):
        hits = O.phrase_search(idx, [0, 1, 2], [0, 0, 0], slop, True, w, cache)
        assert len(hits) == n, slop
        d, s, c = native_batch(index_to_csr(idx), np.array([[0, 1, 2]], np.uint32), np.zeros((1, 3), np.uint32),
                               np.array([slop], np.uint32), [w], cache, True, 4, threads=1)
        assert int(c[0]) == n and (not n or (d[0, 0] == 0 and s[0, 0].view(np.uint32) == hits[0][0].view(np.uint32))), slop
