"""Fixtures for the top-k selection range tests (tests/test_topk_range_{gpu,emulated}.py): posting lists whose postings all
score the same, k values on the candidate-buffer boundaries of every top-k kernel, batches whose heavy query is cut into a
known number of doc ranges, and f64 signal columns / coefficients / boosts that give negative, -0.0, +-inf and NaN totals.
Each builder asserts that it produced its targets.

Buffer sizes restated from bm25.cu (all powers of two):
  k_or3 / k_topk_warp   cap  = max(1024, next >= k + n_terms * 128)
  k_sig_multi           cap  = max(1024, next >= k + n_slots * 128)
  k_plan_recall         rcap = max(1024, next >= k + 32)
  k_wand                wcap = next >= 2k
  k_merge_topk          W <= min(16, 16384 / k) ranges, capm = max(1024, next >= W_max * k)
"""
import struct

import numpy as np

MAX_K = 4096
FIELDNORM_ID = 20                    # every document of a tie index has this fieldnorm code


def next_pow2(x, lo):
    c = lo
    while c < x:
        c <<= 1
    return c


def boundary_ks(n_slots=(1, 2, 8, 16)):
    """k at 1 and the 2^n - 1 / 2^n / 2^n + 1 edges, and for every buffer rule the k that fills it to exactly a power of two
    and the k one above (which doubles it)"""
    ks = {1, 31, 32, 33, 127, 128, 129, 1023, 1024, 1025, 2047, 2048, 4095, 4096}
    for nt in n_slots:                                   # cap = k + nt * 128
        ks |= {4096 - nt * 128, 4096 - nt * 128 + 1}
    ks |= {1024, 1025, 2048, 2049}                       # wcap = 2k
    ks |= {1024 - 32, 1024 - 32 + 1, 4096 - 32, 4096 - 32 + 1}   # rcap = k + 32
    ks = sorted(k for k in ks if 1 <= k <= MAX_K)
    assert {3072, 3073, 3968, 3969, 4064, 4065, 2049} <= set(ks)
    assert next_pow2(3072 + 8 * 128, 1024) == 4096 and next_pow2(3073 + 8 * 128, 1024) == 8192
    return ks


def tie_dfs(ks):
    return sorted({d for k in ks for d in (k - 1, k, k + 1, 2 * k, 2 * k + 1) if d >= 1})


def tie_index(seed, max_doc, ks):
    """term t has doc_freq dfs[t] (k - 1, k, k + 1, 2k, 2k + 1 for every k), tf 1 everywhere, and every document has the
    fieldnorm code FIELDNORM_ID: within a term every posting scores the same f32 value, so the k-th place is always a tie
    decided by doc id.  Returns dict(docs, tfs, ids, dfs)."""
    rng = np.random.default_rng(seed)
    dfs = tie_dfs(ks)
    assert max(dfs) <= max_doc
    docs = [np.sort(rng.choice(max_doc, d, replace=False)).astype(np.uint32) for d in dfs]
    tfs = [np.ones(d, np.uint32) for d in dfs]
    ids = np.full(max_doc, FIELDNORM_ID, np.uint8)
    # self-check: every (k +- 1, 2k, 2k + 1) doc_freq is present, one fieldnorm code and one tf per term
    have = {int(d.size) for d in docs}
    for k in ks:
        assert {k, k + 1, 2 * k, 2 * k + 1} <= have and (k == 1 or k - 1 in have), k
    assert all(np.all(t == 1) for t in tfs) and np.unique(ids).size == 1
    return dict(docs=docs, tfs=tfs, ids=ids, dfs=dfs)


def term_of_df(fx, df):
    return fx["dfs"].index(df)


# ------------------------------------------------------------------ doc-range splits --------------------------------------
def plan_w(work, k, can_split=True):
    """plan_items (bm25.cu) restated: the number of doc ranges W of every query, from the queries' posting counts"""
    work = [int(w) for w in work]
    nq = len(work)
    target = max(32768, sum(work) // max(nq, 1))
    wmax = max(1, min(16, 16384 // k))
    return [min(wmax, -(-w // target)) if can_split else 1 for w in work]


def range_bounds(max_doc, W):
    """the inner boundaries max_doc * c / W, c = 1..W-1, of a query cut into W ranges"""
    return [max_doc * c // W for c in range(1, W)]


def split_index(seed, max_doc, heavy_dfs, n_light=40, light_df=64):
    """A tie-scored index for split batches: heavy terms of the given doc_freqs, a `boundary` term per heavy term that holds
    the documents max_doc*c/W - 1, max_doc*c/W and max_doc*c/W + 1 for the W that heavy term gets (and every other W up to
    16), and light terms.  Query (heavy, boundary) in OR or AND ranks the boundary documents first, all with one score,
    so equal scores straddle every range boundary.  Returns dict(docs, tfs, ids, heavy, boundary, light)."""
    rng = np.random.default_rng(seed)
    edge = sorted({b + o for W in range(2, 17) for b in range_bounds(max_doc, W) for o in (-1, 0, 1)})
    edge = np.array(edge, np.uint32)
    docs, heavy, boundary = [], [], []
    for df in heavy_dfs:
        rest = np.setdiff1d(np.arange(max_doc, dtype=np.uint32), edge)
        d = np.union1d(edge, rng.choice(rest, df - edge.size, replace=False)).astype(np.uint32)
        assert d.size == df
        heavy.append(len(docs)); docs.append(d)
        boundary.append(len(docs)); docs.append(edge.copy())
    light = []
    for _ in range(n_light):
        light.append(len(docs)); docs.append(np.sort(rng.choice(max_doc, light_df, replace=False)).astype(np.uint32))
    tfs = [np.ones(d.size, np.uint32) for d in docs]
    return dict(docs=docs, tfs=tfs, ids=np.full(max_doc, FIELDNORM_ID, np.uint8), heavy=heavy, boundary=boundary, light=light,
                edge=edge, max_doc=max_doc)


def split_batch(fx, h, n_light=None):
    """rows [nq, 2]: query 0 = (heavy h, its boundary term), the others (light, NO_TERM)"""
    NO_TERM = 0xFFFFFFFF
    light = fx["light"][:n_light]
    rows = np.full((1 + len(light), 2), NO_TERM, np.uint32)
    rows[0] = [fx["heavy"][h], fx["boundary"][h]]
    rows[1:, 0] = light
    return rows


def work_of(fx, rows):
    return [sum(int(fx["docs"][t].size) for t in r if t != 0xFFFFFFFF) for r in rows]


# ------------------------------------------------------------------ f64 special values ------------------------------------
F64_MAX = np.finfo(np.float64).max
SUB = 5e-324
NAN_P = struct.unpack("<d", struct.pack("<Q", 0x7FF8000000000000))[0]
NAN_N = struct.unpack("<d", struct.pack("<Q", 0xFFF8000000000000))[0]
SPECIAL = np.array([-1.5, -0.0, 0.0, SUB, -SUB, F64_MAX, -F64_MAX, np.inf, -np.inf, NAN_P, NAN_N, 2.0, -2.0, 1.0, 3.0, -3.0],
                   np.float64)


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def special_columns(max_doc, seed):
    """col 0 cycles through SPECIAL (so every value, NaNs of both signs included, recurs and ties); col 1 holds small
    integers (exact sums, more ties) and +-inf on a few docs; col 2 is -(doc id) (a strict order that falls with the doc)"""
    rng = np.random.default_rng(seed)
    c0 = SPECIAL[np.arange(max_doc) % SPECIAL.size].copy()
    c1 = rng.integers(-3, 4, max_doc).astype(np.float64)
    c1[rng.choice(max_doc, 8, replace=False)] = np.inf
    c1[rng.choice(max_doc, 8, replace=False)] = -np.inf
    c2 = -np.arange(max_doc, dtype=np.float64)
    b0 = bits(c0)
    assert np.signbit(c0[np.isnan(c0)]).any() and (~np.signbit(c0[np.isnan(c0)])).any()   # NaNs of both signs
    assert (b0 == 0x8000000000000000).any() and (b0 == 0).any() and (b0 == 1).any() and (b0 == 0x8000000000000001).any()
    return [c0, c1, c2]


def canon(x):
    """the library's NaN rule: every NaN total is the negative quiet NaN 0xFFF8000000000000"""
    x = np.array(x, np.float64)
    x[np.isnan(x)] = NAN_N
    return x


def order_key(x):
    """f64::total_cmp over canon(x), as an int (bigger ranks first)"""
    b = int(bits(canon([x]))[0])
    return b ^ 0xFFFFFFFFFFFFFFFF if b >> 63 else b | 0x8000000000000000


def expected_topk(totals, docs, k):
    """(total desc by order_key, doc asc) top k over a plain list"""
    o = sorted(range(len(docs)), key=lambda i: (-order_key(totals[i]), int(docs[i])))[:k]
    return np.array([docs[i] for i in o], np.uint32), np.array([totals[i] for i in o], np.float64)


def same_totals(a, b):
    """bit-equal, with any NaN equal to any NaN"""
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(bits(a)[~na], bits(b)[~nb]))
