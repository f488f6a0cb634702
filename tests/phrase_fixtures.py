"""Shared helpers of the phrase-query tests, smoke() and tools/phrase_bench.py (no pytest import): an oracle index as a
device segment, a random token-stream index, the oracle's answer for a batch, the bit-level comparison, and the native
threaded oracle (phrase_oracle_mt.cpp) compiled into a temporary directory."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import phrase_oracle as O

def make_segment(index, **kw):
    """An oracle index as a device segment with record option 2 and its positions attached."""
    from stract_b200.bm25 import SegmentReader, encode_positions, encode_postings
    terms = index["terms"]
    ids = index["fieldnorm_ids"]
    n = ids.size
    avg = np.float32(np.float32(index["total_num_tokens"]) / np.float32(n))
    tfs = [np.array([len(p) for p in t["positions"]], np.uint32) for t in terms]
    data, infos = encode_postings([t["docs"] for t in terms], tfs, ids, avg, record_option=2)
    off = np.concatenate([[0], np.cumsum([len(t["docs"]) for t in terms])])
    flat = [p for t in terms for p in t["positions"]]
    pos, po, pl = encode_positions(np.concatenate(flat) if flat else np.zeros(0, np.uint32), np.concatenate(tfs), off)
    return SegmentReader(data, infos, ids, record_option=2, total_num_tokens=index["total_num_tokens"], positions=pos,
                         positions_ranges=(po, pl), **kw)


def random_index(seed, n_docs, n_vocab=24, long_doc=3000):
    """Token streams from a Zipf vocabulary (phrases occur by chance), lengths LogNormal; term n_vocab appears in exactly 256
    docs, term n_vocab+1 in 50 (vint-only), and doc 0 alternates terms 0 and 1 `long_doc` times (a tf above the shared
    buffer, positions over many blocks)."""
    from stract_b200.bm25 import fieldnorm_table, fieldnorms_to_ids
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, n_vocab + 1) ** 1.1
    p /= p.sum()
    lens = np.clip(rng.lognormal(2.8, 0.8, n_docs), 2, 400).astype(np.int64)
    lens[0] = long_doc
    special = {n_vocab: set(rng.choice(np.arange(1, n_docs), 256, replace=False).tolist()),
               n_vocab + 1: set(rng.choice(np.arange(1, n_docs), 50, replace=False).tolist())}
    post = {}
    for d in range(n_docs):
        toks = (np.arange(long_doc) % 2) if d == 0 else rng.choice(n_vocab, lens[d], p=p)
        toks = np.array(toks)
        for s, docs in special.items():
            if d in docs:
                toks[rng.integers(0, len(toks))] = s
        for t in np.unique(toks):
            post.setdefault(int(t), {})[d] = np.flatnonzero(toks == t).astype(np.uint32)
    terms = []
    for t in range(n_vocab + 2):
        ds = sorted(post.get(t, {}))
        terms.append({"docs": np.array(ds, np.uint32), "positions": [post[t][d] for d in ds]})
    ids = fieldnorms_to_ids(lens.astype(np.uint32))
    total = int(fieldnorm_table()[ids].astype(np.uint64).sum())
    return {"fieldnorm_ids": ids, "terms": terms, "total_num_tokens": total}, rng


def oracle_batch(index, rows, offsets, slops, scoring, k, total_docs=None, avg=None, dfs=None):
    """The oracle's answer for every row (ABSENT / NO_TERM handled like the library)."""
    from stract_b200.bm25 import ABSENT_TERM, NO_TERM
    n = index["fieldnorm_ids"].size
    total_docs = n if total_docs is None else total_docs
    avg = np.float32(np.float32(index["total_num_tokens"]) / np.float32(n)) if avg is None else avg
    cache = O.tf_cache(avg, [__import__("stract_b200.bm25", fromlist=["x"]).id_to_fieldnorm(i) for i in range(256)])
    out = []
    for q in range(rows.shape[0]):
        real = [j for j in range(rows.shape[1]) if rows[q, j] != NO_TERM]
        terms = [None if rows[q, j] == ABSENT_TERM else int(rows[q, j]) for j in real]
        df = [0 if t is None else len(index["terms"][t]["docs"]) for t in terms] if dfs is None else list(dfs[q])
        w = O.bm25_weight_for_terms(df, total_docs)
        out.append(O.phrase_search(index, terms, [int(offsets[q, j]) for j in real], int(slops[q]), scoring, w, cache, k))
    return out


def assert_same(got, want):
    d, s, n = got
    for q, hits in enumerate(want):
        assert int(n[q]) == len(hits), (q, int(n[q]), len(hits))
        assert np.array_equal(d[q, :n[q]], np.array([h[1] for h in hits], np.uint32)), q
        assert np.array_equal(s[q, :n[q]].view(np.uint32), np.array([h[0] for h in hits], np.float32).view(np.uint32)), q


def random_rows(rng, n_vocab, nq, width, absent=True):
    from stract_b200.bm25 import ABSENT_TERM, NO_TERM
    p = 1.0 / np.arange(1, n_vocab + 3) ** 0.6
    p /= p.sum()
    rows = np.full((nq, width), NO_TERM, np.uint32); offs = np.zeros((nq, width), np.uint32)
    for q in range(nq):
        m = int(rng.integers(2, width + 1))
        rows[q, :m] = rng.choice(n_vocab + 2, m, p=p)
        if rng.random() < 0.3:
            rows[q, 1] = rows[q, 0]                        # a duplicate term: two cursors
        gaps = rng.integers(1, 3, m) if rng.random() < 0.3 else np.ones(m, np.int64)
        offs[q, :m] = np.cumsum(gaps) - gaps[0]            # non-trivial offsets, in offset order
        if absent and rng.random() < 0.05:
            rows[q, m - 1] = ABSENT_TERM
    return rows, offs

_NATIVE = None


def native_oracle():
    """phrase_oracle_mt.cpp compiled with g++ into a temporary directory (nothing is written to the tree), loaded once."""
    global _NATIVE
    if _NATIVE is None:
        src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "phrase_oracle_mt.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="phrase_oracle_"), "libphrase_oracle.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-pthread",
                               src, "-o", out])
        L = C.CDLL(out)
        L.phrase_oracle_batch.restype = C.c_int
        _NATIVE = L
    return _NATIVE


def native_batch(csr, rows, offsets, slops, weights, cache, scoring, k, threads):
    """The native oracle over an index in CSR form (dict: docs, term_off, positions, pos_off, fieldnorm_ids): one query per
    host thread.  Returns (docs [nq,k], scores [nq,k], n [nq])."""
    L = native_oracle()
    rows = np.ascontiguousarray(rows, np.uint32); offs = np.ascontiguousarray(offsets, np.uint32)
    sl = np.ascontiguousarray(slops, np.uint32); w = np.ascontiguousarray(weights, np.float32)
    cache = np.ascontiguousarray(cache, np.float32)
    nq, nt = rows.shape
    d = np.zeros((nq, k), np.uint32); s = np.zeros((nq, k), np.float32); n = np.zeros(nq, np.uint32)
    a = [np.ascontiguousarray(csr[x]) for x in ("docs", "term_off", "positions", "pos_off", "fieldnorm_ids")]
    P = lambda x: C.c_void_p(x.ctypes.data)
    rc = L.phrase_oracle_batch(P(a[0]), P(a[1]), C.c_uint32(a[1].size - 1), P(a[2]), P(a[3]), P(a[4]), P(cache), C.c_uint32(nq),
                               C.c_uint32(nt), P(rows), P(offs), P(sl), P(w), C.c_int(1 if scoring else 0), C.c_uint32(k), P(d), P(s),
                               P(n), C.c_int(threads))
    assert rc == 0, "native oracle: term id out of range"
    return d, s, n


def index_to_csr(index):
    """An oracle index (per-term dicts) in the CSR form native_batch takes."""
    terms = index["terms"]
    term_off = np.concatenate([[0], np.cumsum([len(t["docs"]) for t in terms])]).astype(np.uint64)
    flat = [p for t in terms for p in t["positions"]]
    pos_off = np.concatenate([[0], np.cumsum([len(p) for p in flat])]).astype(np.uint64)
    return {"docs": np.concatenate([t["docs"] for t in terms]).astype(np.uint32), "term_off": term_off,
            "positions": np.concatenate(flat).astype(np.uint32), "pos_off": pos_off,
            "fieldnorm_ids": np.ascontiguousarray(index["fieldnorm_ids"], np.uint8)}
