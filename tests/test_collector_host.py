"""BucketCollector mirror (stract_b200/collector.py) pinned on the reference's own scenarios
(crates/core/src/collector/top_docs.rs:493-751), and the top-K harvest against the insert-everything harvest."""
import numpy as np

from stract_b200.collector import BucketCollector, CollectorConfig, Hashes, SimhashTable, harvest_top_k


def run(top_n, docs):
    c = BucketCollector(top_n, CollectorConfig())
    for (site, title, url, uwt, sim), doc, score in docs:
        c.insert(score, Hashes(site, title, url, uwt, sim), (score, doc))
    return c.into_sorted_vec(True)


def test_all_different():        # top_docs.rs:518-583
    docs = [((i, i, i, i, s), 122 + i, float(i)) for i, s in zip(range(1, 6), (12, 123, 1234, 12345, 123456))]
    assert run(3, docs) == [(5.0, 127), (4.0, 126), (3.0, 125)]


def test_less_than_topn():       # top_docs.rs:585-627
    docs = [((3, 3, 3, 3, 12), 125, 3.0), ((4, 4, 4, 4, 123), 126, 4.0), ((5, 5, 5, 5, 1234), 127, 5.0)]
    assert run(10, docs) == [(5.0, 127), (4.0, 126), (3.0, 125)]


def test_same_key_de_prioritised():   # top_docs.rs:629-705
    docs = [((1, 1, 1, 1, 12), 125, 3.0), ((2, 2, 2, 2, 123), 126, 3.1), ((2, 2, 2, 2, 1234), 127, 5.0)]
    assert run(10, docs) == [(5.0, 127), (3.0, 125), (3.1, 126)]
    assert run(2, docs) == [(5.0, 127), (3.0, 125)]


def test_simhash_dedup():        # top_docs.rs:707-750
    docs = [((1, 1, 1, 1, 1234), 125, 3.0), ((2, 2, 2, 2, 1234), 126, 3.1), ((3, 3, 3, 3, 1), 127, 5.0)]
    assert run(10, docs) == [(5.0, 127), (3.1, 126), (3.0, 125)]


def test_simhash_table_is_hamming_ball():   # simhash.rs:69-135: K = 3
    t = SimhashTable()
    t.insert(0b1111_0000)
    assert t.contains(0b1111_0000) and t.contains(0b1111_0111) and not t.contains(0b1111_1111 ^ 0b1111_0000 ^ 0b1_0000_0000)


def test_harvest_over_top_k_equals_harvest_over_everything():
    rng = np.random.default_rng(3)
    for trial in range(20):
        n = 5000
        totals = rng.random(n) ** 3 * 10.0
        site = rng.integers(0, 40 if trial % 2 else 2000, n)      # few sites: heavy de-ranking, K has to grow
        url = rng.integers(0, 1 << 40, n); title = rng.integers(0, 3000, n) + (1 << 41)
        sim = rng.integers(1, 1 << 62, n)
        hashes = [Hashes(int(site[i]) + (1 << 50), int(title[i]), int(url[i]), int(url[i]) ^ 1, int(sim[i])) for i in range(n)]
        order = np.lexsort((np.arange(n), -totals))

        def search(K):
            return order[:K], totals[order[:K]]
        top_n = 100
        full = BucketCollector(top_n, CollectorConfig())
        for d in order:                      # the reference's collector sees every document (ascending doc order there;
            full.insert(float(totals[d]), hashes[d], (int(d), float(totals[d])))   # scores are distinct, order is immaterial)
        want = full.into_sorted_vec(True)
        got, K, proven = harvest_top_k(top_n, search, lambda d: hashes[d], k_max=8192)
        assert proven and got == want, (trial, K)


def test_total_cmp_order_of_negative_zero_and_infinite_scores():
    """ScoredDoc::cmp is f64::total_cmp (top_docs.rs:229-233): -0.0 pops after +0.0, -inf last, +inf first"""
    scores = [-1.5, 0.0, -0.0, np.inf, -np.inf, 2.0, -3.0, 5e-324, -5e-324]
    docs = [((i + 1, 100 + i, 200 + i, 300 + i, 0), i, s) for i, s in enumerate(scores)]
    got = [s for s, _ in run(len(scores), docs)]
    want = [np.inf, 2.0, 5e-324, 0.0, -0.0, -5e-324, -1.5, -3.0, -np.inf]
    assert [np.float64(x).view(np.uint64) for x in got] == [np.float64(x).view(np.uint64) for x in want]


def test_negative_scores_are_de_ranked_by_the_adjuster():
    """the penalty divides the score, so a negative score moves UP towards 0 when its site was picked, as in the reference"""
    c = BucketCollector(3, CollectorConfig())
    for site, doc, score in ((1, 0, 0.5), (1, 1, -0.9), (2, 2, -0.95)):
        c.insert(score, Hashes(site, 10 + doc, 20 + doc, 30 + doc, 0), doc)
    got = c.into_sorted_vec(True, with_adjusted=True)
    assert [d for d, _ in got] == [0, 1, 2] and got[1][1] == -0.9 * (1.0 / 1.1) and got[2][1] == -0.95


def test_nan_scores_rank_by_their_bits_and_terminate():
    """a positive NaN pops before +inf, a negative NaN after -inf; and after a pick the loop that re-adjusts the best
    document meets a NaN at the top (the second positive NaN) and ends, because it compares bits -- the reference's `==`
    never holds for a NaN and would loop forever"""
    import struct
    import threading
    pos = struct.unpack("<d", struct.pack("<Q", 0x7FF8000000000000))[0]
    neg = struct.unpack("<d", struct.pack("<Q", 0xFFF8000000000000))[0]
    docs = [((1, 10, 20, 30, 0), 0, neg), ((1, 11, 21, 31, 0), 1, 1.0), ((2, 12, 22, 32, 0), 2, pos), ((3, 13, 23, 33, 0), 3, -np.inf),
            ((4, 14, 24, 34, 0), 4, np.inf), ((5, 15, 25, 35, 0), 5, pos)]
    out = []
    t = threading.Thread(target=lambda: out.append(run(6, docs)), daemon=True)
    t.start(); t.join(30)
    assert out, "the collector did not terminate on a NaN best document"
    assert [d for _, d in out[0]] == [2, 5, 4, 1, 3, 0]
