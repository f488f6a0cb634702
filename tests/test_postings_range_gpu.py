"""The BM25 device decoders over the posting format's full value range (fixtures: tests/postings_range.py).  Needs a GPU.

Every kernel that reads tantivy's posting format decodes blocks of 0..31-bit doc deltas and 0..32-bit tfs, VInt tails with
1- to 5-byte values, block-wand tf code 255 (saturated) and all 256 fieldnorm codes here, on a medium index (~2^22 docs,
both record options) and on one at the largest max_doc the library accepts (2^31 - 2).  Bar: bit-exact against the
oracle, and, where the oracle would only decode the same bytes again, against the input: a single-term query with
k >= df returns exactly the input docs with scores equal to a vectorised f32 restatement of Bm25Weight.score, and docsets
read back the input docs."""
import resource
import time

import numpy as np
import pytest

import postings_range as R
import test_bm25_gpu as T
from stract_b200 import bm25
from stract_b200.bm25 import MODE_AND, MODE_OR, MODE_OR_WAND, NO_TERM, Docset, SegmentReader, TopDocs

pytestmark = pytest.mark.gpu

MEDIUM = (1 << 22) + 12_345
NEAR_LIMIT = (1 << 31) - 2   # the largest max_doc below TERMINATED: doc ids up to 2^31 - 3
MAX_K = 4096


def make(seed, max_doc, record_option=1, big=True):
    """A range index as oracle Segment + device SegmentReader, after its self-check."""
    fx = R.range_index(seed, max_doc, record_option, big)
    oseg, seg = T.build(fx["docs"], fx["tfs"], None, record_option, fieldnorm_ids=fx["ids"])
    fx["produced"] = R.self_check(fx, oseg.postings_bytes(), oseg.term_infos())
    fx["oseg"], fx["seg"] = oseg, seg
    return fx


def expected_single(fx, t, k):
    """top k of term t alone, from the input (docs, tfs, fieldnorm ids): tantivy's Bm25Weight.score in f32, order
    (score desc, doc asc)"""
    seg = fx["seg"]
    d = fx["docs"][t]
    tf = fx["tfs"][t].astype(np.float32)
    w = np.float32(bm25.Bm25Weight.for_one_term(d.size, seg.max_doc, seg.average_fieldnorm).weight)
    cache = bm25.compute_tf_cache(seg.average_fieldnorm)
    s = (w * (tf / (tf + cache[fx["ids"][d]]))).astype(np.float32)
    o = np.lexsort((d, -s))[:k]
    return d[o], s[o]


def check_single_term_raw(fx, ks=(10, MAX_K)):
    """every term alone in AND (k_and3; k_topk_warp when the batch holds a clause above 65 536 postings) and OR (k_or3):
    docs and score bits from the input, not from the format.  OR_WAND (k_wand) alone against the oracle's walk (mode 1):
    the reference's one-clause walk may skip a tail whose best score lies above Bm25Weight::max_score."""
    seg = fx["seg"]
    nt = seg.n_terms
    small = np.array([t for t in range(nt) if seg.doc_freq[t] <= 65_536], np.uint32)
    batches = [(MODE_AND, small), (MODE_AND, np.arange(nt, dtype=np.uint32)), (MODE_OR, np.arange(nt, dtype=np.uint32)),
               (MODE_OR_WAND, np.arange(nt, dtype=np.uint32))]
    for mode, terms in batches:
        for k in ks:
            gd, gs, gn = TopDocs.with_limit(k).search_batch(seg, terms[:, None], mode)
            for q, t in enumerate(terms):
                if mode == MODE_OR_WAND:
                    ed, es, _ = fx["oseg"].topk(np.array([t], np.uint32), *T.weights_for(seg, [t]), 1, k)
                else:
                    ed, es = expected_single(fx, int(t), k)
                m = int(gn[q])
                assert m == ed.size, (mode, k, int(t), m, ed.size)
                assert np.array_equal(gd[q, :m], ed), (mode, k, int(t))
                assert np.array_equal(gs[q, :m].view(np.uint32), es.view(np.uint32)), (mode, k, int(t))


def _group_queries(fx, rng, nq, width=4):
    """AND queries of 1..4 terms drawn from one group of overlapping terms, padded with NO_TERM"""
    rows = np.full((nq, width), NO_TERM, np.uint32)
    for q in range(nq):
        g = fx["groups"][int(rng.integers(0, len(fx["groups"])))]
        n = int(rng.integers(1, min(width, len(g)) + 1))
        rows[q, :n] = rng.choice(g, n, replace=False)
    return rows


def _against_oracle(fx, rows, mode, omode, k):
    """`omode`: the oracle mode, or a function of the query's clause count that gives it"""
    oseg, seg = fx["oseg"], fx["seg"]
    gd, gs, gn = TopDocs.with_limit(k).search_batch(seg, rows, mode)
    hits = 0
    for q in range(rows.shape[0]):
        qq = np.array([x for x in rows[q] if x != NO_TERM], np.uint32)
        od, os_, _ = oseg.topk(qq, *T.weights_for(seg, qq), omode(qq.size) if callable(omode) else omode, k)
        m = int(gn[q])
        assert m == len(od), (mode, k, q, qq, m, len(od))
        assert np.array_equal(gd[q, :m], od) and np.array_equal(gs[q, :m], os_), (mode, k, q, qq)
        hits += m
    return hits


def check_and(fx, rng, nq, ks=(1, 10, 1000, MAX_K), monkeypatch=None):
    """AND vs oracle mode 0: batches of k_and3 (no clause above 65 536 alone) and of k_topk_warp<AND> (the same queries
    plus the large term alone); again with a 1 MB candidate budget (several candidate groups) when monkeypatch is given.
    One-clause queries are compared with the exhaustive oracle (mode 2): the reference runs them through
    block_wand_single_scorer, which bounds a VInt tail it has not loaded by Bm25Weight::max_score, and that is below the
    score of a tail posting with a tf in the hundreds of thousands on a short document (the large term has one), so at
    k = 1 the reference can skip the tail's best doc.  The library's AND is exact; OR_WAND keeps the reference's walk."""
    seg = fx["seg"]
    rows = _group_queries(fx, rng, nq)
    single_big = (rows[:, 1] == NO_TERM) & (seg.doc_freq[rows[:, 0]] > 65_536)
    rows = rows[~single_big]
    big = [t for t in range(seg.n_terms) if seg.doc_freq[t] > 65_536]
    batches = [rows] + [np.vstack([rows, np.array([[t] + [NO_TERM] * 3], np.uint32)]) for t in big[:1]]
    budgets = (None, "1") if monkeypatch is not None else (None,)
    for budget in budgets:
        if budget:
            monkeypatch.setenv("SB200_AND3_BUDGET_MB", budget)
        for b in batches:
            for k in ks:
                assert _against_oracle(fx, b, MODE_AND, lambda n: 0 if n > 1 else 2, k) > 0
    if monkeypatch is not None:
        monkeypatch.delenv("SB200_AND3_BUDGET_MB")


def check_or(fx, rng, nq, ks, sig_nq, sig_k, sig_cols=(4, 2, 0), sig_max_docs=(0, 137)):
    """OR through k_or3 (staged and direct blocks, doc-range items, NO_TERM pads) vs the exhaustive union, and the signal
    combine (k_or3<SIGNAL>, k_topk_warp for the max_docs cut) vs the oracle"""
    T.union_kernel_check(fx["oseg"], fx["seg"], rng, nq, ks, 5, sig_nq, sig_k, sig_cols, sig_max_docs)


def check_wand(fx, rng, nq, ks=(1, 10, 300)):
    """OR_WAND (k_wand) vs the oracle's block_wand: random 1..8-term queries, group queries, and the saturation term,
    whose blocks' best postings (tf 254, 255, 256, ... 10^8 on one-token docs) score higher block after block: a block
    bound computed from tf 255 instead of u32::MAX would skip them"""
    seg = fx["seg"]
    for width in (1, 2, 3, 5, 8):
        rows = np.stack([rng.choice(seg.n_terms, width, replace=False) for _ in range(nq)]).astype(np.uint32)
        for k in ks:
            _against_oracle(fx, rows, MODE_OR_WAND, 1, k)
    for k in ks:
        _against_oracle(fx, _group_queries(fx, rng, nq), MODE_OR_WAND, 1, k)
    for s in fx["saturated"]:
        g = next(g for g in fx["groups"] if s in g)
        rows = np.array([[s, NO_TERM], g[:2]], np.uint32)
        for k in (1, 2, 5):
            _against_oracle(fx, rows, MODE_OR_WAND, 1, k)
        d, _, n = TopDocs.with_limit(1).search_batch(seg, rows[:1], MODE_OR_WAND)
        assert n[0] == 1 and fx["tfs"][s][np.searchsorted(fx["docs"][s], d[0, 0])] == R.SATURATED[-1]
    # one-clause walks that leave a block unloaded: the tail of tail_max (and of the large term) is bounded by max_score
    # and skipped by the reference at small k; the first assertion shows the fixture reaches that case
    t = fx["tail_max"][0]
    od, _, _ = fx["oseg"].topk(np.array([t], np.uint32), *T.weights_for(seg, [t]), 1, 1)
    assert od[0] != expected_single(fx, t, 1)[0][0], "the reference's one-clause walk no longer skips the tail"
    big = [x for x in range(seg.n_terms) if seg.doc_freq[x] > 65_536]
    rows = np.array([[x] for x in fx["tail_max"] + big], np.uint32)
    for k in (1, 2, 3, 10):
        _against_oracle(fx, rows, MODE_OR_WAND, 1, k)


def check_docsets(fx):
    """Docset.from_postings reads back every term's input docs; an AND of two overlapping terms is their intersection"""
    seg = fx["seg"]
    for t in range(seg.n_terms):
        ds = Docset.from_postings(seg, t)
        assert ds.count() == fx["docs"][t].size, t
        assert np.array_equal(ds.docs(), fx["docs"][t]), t
        ds.close()
    for g in fx["groups"]:
        a, b = Docset.from_postings(seg, g[0]), Docset.from_postings(seg, g[-1])
        c = Docset.combine("and", [a, b])
        assert np.array_equal(c.docs(), np.intersect1d(fx["docs"][g[0]], fx["docs"][g[-1]])), g
        for x in (a, b, c):
            x.close()


def check_max_doc_limit():
    """max_doc = 2^31 - 1 (TERMINATED) is refused with SB200_ERANGE before anything is read or allocated"""
    from stract_b200._lib import Sb200Error
    ids = np.zeros((1 << 31) - 1, np.uint8)   # calloc'd: its pages are never touched
    with pytest.raises(Sb200Error) as e:
        SegmentReader(np.zeros(1, np.uint8), (np.zeros(0), np.zeros(0), np.zeros(0)), ids, total_num_tokens=0)
    assert e.value.code == -4   # SB200_ERANGE


@pytest.fixture(scope="module")
def medium():
    return make(41, MEDIUM)


def test_medium_self_check_and_raw_single_terms(medium):
    check_single_term_raw(medium)


def test_medium_and(medium, monkeypatch):
    check_and(medium, np.random.default_rng(1), 120, monkeypatch=monkeypatch)


def test_medium_or_and_signals(medium):
    check_or(medium, np.random.default_rng(2), 60, (1, 10, 1000), 40, 1000)


def test_medium_or_wand(medium):
    check_wand(medium, np.random.default_rng(3), 16)


def test_medium_docsets(medium):
    check_docsets(medium)


def test_medium_record_option_2():
    fx = make(43, MEDIUM, record_option=2)
    rng = np.random.default_rng(4)
    check_single_term_raw(fx)
    check_and(fx, rng, 60, ks=(10, MAX_K))
    check_or(fx, rng, 30, (10, 1000), 20, 500, sig_cols=(2,))
    check_wand(fx, rng, 8, ks=(10,))


def test_max_doc_limit_refused():
    check_max_doc_limit()


def test_near_limit_index():
    """max_doc = 2^31 - 2: 24- and 31-bit doc deltas, 5-byte VInt gaps, doc ids up to 2^31 - 3.  No signal columns
    (17 GB of f64).  Prints the time of each stage and the peak host memory."""
    t0 = time.time()
    fx = make(47, NEAR_LIMIT)
    assert {24, 31} <= fx["produced"]["wd"] and 5 in fx["produced"]["gap_bytes"]
    stages = [("build", time.time() - t0)]
    rng = np.random.default_rng(5)
    for name, f in (("raw", lambda: check_single_term_raw(fx)), ("and", lambda: check_and(fx, rng, 60, ks=(10, MAX_K))),
                    ("or", lambda: check_or(fx, rng, 24, (10, 1000), 0, 0, sig_cols=())),
                    ("wand", lambda: check_wand(fx, rng, 8, ks=(10,))), ("docsets", lambda: check_docsets(fx))):
        t = time.time()
        f()
        stages.append((name, time.time() - t))
    print("near-limit index:", ", ".join(f"{n} {s:.1f} s" for n, s in stages),
          f"; peak host RSS {resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20:.2f} GB")


def check_positions(seed=51):
    """k_positions_read reads back the input position deltas of wide blocks (widths 0..31), a VInt tail with 1- to 5-byte
    deltas and a posting of tf 2^16 + 1, whole and in windows that start and end inside blocks and the tail"""
    import phrase_fixtures
    from stract_b200.bm25 import encode_positions
    index, deltas = R.positions_index(seed)
    tfs = np.concatenate([[len(p) for p in t["positions"]] for t in index["terms"]]).astype(np.uint32)
    off = np.cumsum([0] + [len(t["docs"]) for t in index["terms"]])
    pos, po, pl = encode_positions(np.concatenate([p for t in index["terms"] for p in t["positions"]]), tfs, off)
    widths, lens = R.parse_positions(pos, po[0], pl[0])
    assert set(widths) == set(R.PW) and set(lens) >= {1, 2, 3, 4, 5}, (widths, lens)   # self-check
    assert max(R.parse_positions(pos, po[1], pl[1])[0]) >= 1 and max(tfs) == R.TF16 + 1
    seg = phrase_fixtures.make_segment(index)
    rng = np.random.default_rng(seed)
    for t, d in enumerate(deltas):
        assert np.array_equal(seg.read_positions(t, 0, d.size), d), t
        for _ in range(40):
            a = int(rng.integers(0, d.size)); n = int(rng.integers(1, d.size - a + 1))
            assert np.array_equal(seg.read_positions(t, a, n), d[a:a + n]), (t, a, n)
        for a in range(max(0, d.size - 140), d.size):   # every start in the last block and the tail
            assert np.array_equal(seg.read_positions(t, a, d.size - a), d[a:]), (t, a)


def test_positions_read_back():
    check_positions()

