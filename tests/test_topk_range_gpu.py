"""The top-k selection and the f64 score combine over the score's full range (fixtures: tests/topk_range.py).  Needs a GPU.

Every ranked result goes through one selection: a score becomes an order-preserving key (ord_f32 / ord_f64 with ~doc as
the tie-break), candidates gather in a power-of-two buffer that is re-sorted when the next round would overflow it, and a
query larger than the batch average is cut into doc ranges whose partial lists k_merge_topk merges.  Here that selection
meets k on every buffer boundary with exact ties at the k-th place, split batches whose equal-score documents straddle
the range boundaries, and totals that are negative, -0.0, +-inf and NaN.  Bar: docs, order and score / total bits equal to
the oracle (NaN totals: any NaN equals any NaN; the library hands them over as 0xFFF8000000000000), and where the input
decides the answer, equal to the input."""
import resource
import time

import numpy as np
import pytest

import oracle
import test_bm25_gpu as T
import topk_range as R
from stract_b200 import bm25
from stract_b200.bm25 import (MODE_AND, MODE_OR, MODE_OR_WAND, NO_TERM, MultiFieldSignalComputer, SignalComputer, SignalTable,
                              TopDocs)

pytestmark = pytest.mark.gpu

GPU_MAX_DOC = 300_000
SPLIT_MAX_DOC = 1 << 21
W16_DF = 16 * 32768 - 2048      # heavy term of a W = 16 query (with its boundary term above 15 * 32768 postings)
W2_DF = 50_000


def make_tie(seed, max_doc, ks):
    fx = R.tie_index(seed, max_doc, ks)
    fx["oseg"], fx["seg"] = T.build(fx["docs"], fx["tfs"], None, fieldnorm_ids=fx["ids"])
    return fx


def _compare(gd, gs, gn, rows, oseg, seg, omode, k, tag):
    for q in range(rows.shape[0]):
        qq = np.array([x for x in rows[q] if x != NO_TERM], np.uint32)
        od, os_, _ = oseg.topk(qq, *T.weights_for(seg, qq), omode, k)
        m = int(gn[q])
        assert m == od.size, (tag, k, q, m, od.size)
        assert np.array_equal(gd[q, :m], od), (tag, k, q)
        assert np.array_equal(gs[q, :m].view(np.uint32), os_.view(np.uint32)), (tag, k, q)


def check_boundary_k(fx, ks):
    """AND (k_and3), OR (k_or3) and OR_WAND (k_wand) at every k over the terms of doc_freq k - 1 .. 2k + 1: one-clause
    batches (n_terms 1) give the input's first min(k, df) docs with one score; two-clause batches (n_terms 2, the cap one
    step up) match the oracle.  (k_topk_warp<AND> runs in the split batches.)"""
    seg, oseg = fx["seg"], fx["oseg"]
    for k in ks:
        dfs = [d for d in (k - 1, k, k + 1, 2 * k, 2 * k + 1) if d >= 1]
        one = np.array([[R.term_of_df(fx, d)] for d in dfs], np.uint32)
        for mode, omode in ((MODE_AND, 2), (MODE_OR, 2), (MODE_OR_WAND, 1)):
            gd, gs, gn = TopDocs.with_limit(k).search_batch(seg, one, mode)
            for q, d in enumerate(dfs):
                m = min(k, d)
                assert int(gn[q]) == m, (mode, k, d, int(gn[q]))
                assert np.array_equal(gd[q, :m], fx["docs"][one[q, 0]][:m]), (mode, k, d)
                assert np.unique(gs[q, :m].view(np.uint32)).size == 1, (mode, k, d)
            _compare(gd, gs, gn, one, oseg, seg, omode, k, ("one", mode))
        two = np.array([[R.term_of_df(fx, 2 * k + 1), R.term_of_df(fx, k + 1)], [R.term_of_df(fx, k), R.term_of_df(fx, 2 * k)]], np.uint32)
        for mode, omode in ((MODE_AND, 0), (MODE_OR, 2), (MODE_OR_WAND, 1)):
            gd, gs, gn = TopDocs.with_limit(k).search_batch(seg, two, mode)
            _compare(gd, gs, gn, two, oseg, seg, omode, k, ("two", mode))


def check_k_refused(fx):
    """k = 0 and k = 4097 are refused with SB200_ERANGE by the BM25, signal and multi-field entry points"""
    from stract_b200._lib import Sb200Error
    seg = fx["seg"]
    rows = np.zeros((1, 1), np.uint32)
    for k in (0, R.MAX_K + 1):
        td = TopDocs(1); td.limit = k
        for call in (lambda: td.search_batch(seg, rows, MODE_OR), lambda: SignalComputer(seg, None, ()).top_docs_batch(rows, k),
                     lambda: _multi(fx, None, {}).top_docs_batch(np.zeros((1, 1), np.uint8), rows, k)):
            with pytest.raises(Sb200Error) as e:
                call()
            assert e.value.code == -4, k


COEFFS = [  # (coeff_text, per-column coefficients): negative text coefficients, negative / -0.0 / tiny column ones
    (-0.005, [1.0, 1.0, 0.0]),
    (0.5, [-2.0, -0.0, 1e-300]),
    (-0.0, [-1.0, 0.25, -1.0]),
]


def _signal_rows(fx, k):
    return np.array([[R.term_of_df(fx, 2 * k + 1), R.term_of_df(fx, k)], [R.term_of_df(fx, k + 1), NO_TERM],
                     [R.term_of_df(fx, 2 * k), R.term_of_df(fx, max(1, k - 1))]], np.uint32)


def check_signals(fx, ks, cols, max_docs_list=(0, 137)):
    """SignalComputer.top_docs_batch (k_or3 MODE 2, k_topk_warp MODE 2 with max_docs) over the special columns: totals that
    are negative, +-inf, NaN (inf - inf, 0 * inf, NaN columns) and tie exactly, against the oracle"""
    seg, oseg = fx["seg"], fx["oseg"]
    table = SignalTable(cols)
    cache = bm25.compute_tf_cache(seg.average_fieldnorm)
    seen = dict(nan=0, neg=0, inf=0, ties=0)
    for coeff_text, coeffs in COEFFS:
        comp = SignalComputer(seg, table, coeffs, coeff_text=coeff_text)
        for k in ks:
            rows = _signal_rows(fx, k)
            w = np.array([[bm25.StractBm25Weight.for_one_term(int(seg.doc_freq[t]) if t != NO_TERM else 1, seg.max_doc,
                                                                seg.average_fieldnorm).weight for t in r] for r in rows], np.float32)
            for max_docs in max_docs_list:
                gd, gt, gn = comp.top_docs_batch(rows, k, max_docs=max_docs)
                for q in range(rows.shape[0]):
                    qq = np.array([x for x in rows[q] if x != NO_TERM], np.uint32)
                    od, ot, _ = oseg.signal_topk(qq, w[q, :qq.size], np.tile(cache, (qq.size, 1)), 1.2, coeff_text, cols, coeffs, k,
                                                 max_docs=max_docs)
                    m = int(gn[q])
                    assert m == od.size, (coeff_text, k, max_docs, q)
                    assert np.array_equal(gd[q, :m], od), (coeff_text, k, max_docs, q)
                    assert R.same_totals(gt[q, :m], ot), (coeff_text, k, max_docs, q)
                    t = gt[q, :m]
                    assert np.all(R.bits(t[np.isnan(t)]) == 0xFFF8000000000000)
                    seen["nan"] += int(np.isnan(t).sum()); seen["neg"] += int((t < 0).sum()); seen["inf"] += int(np.isinf(t).sum())
                    seen["ties"] += int(m - np.unique(R.bits(t)).size)
    assert all(v > 0 for v in seen.values()), seen


def _multi(fx, cols, coefficients, numeric=()):
    fields = {"Title": fx["seg"], "CleanBody": fx["seg"]}
    return MultiFieldSignalComputer(fields, {"Bm25Title", "Bm25CleanBody", "TitleCoverage"}, SignalTable(cols) if cols else None,
                                    numeric, coefficients=coefficients)


def multi_vs_oracle(comp, oseg, cols, sf, st, k, boost=None):
    docs, totals, n_out = comp.top_docs_batch(sf, st, k, slot_boost=boost)
    names = comp.names
    caches = comp.last_inputs["caches"]
    coefs = [np.float32(comp.field_coefficient(n)) for n in names]
    ops = [(kind, names.index(field) if field is not None else 0, chain, col, comp.coefficient(name, coef))
           for name, kind, field, chain, col, coef in comp.order.entries]
    for q in range(sf.shape[0]):
        od, ot = oracle.multi_signal_topk([oseg] * len(names), caches, [1.2] * len(names), coefs, sf[q], st[q], comp.last_inputs["idf"][q],
                                          comp.last_inputs["idf_f"][q], ops, cols, k, None if boost is None else boost[q])
        n = int(n_out[q])
        assert n == od.size, (q, k, n, od.size)
        assert np.array_equal(docs[q, :n], od), (q, k)
        assert R.same_totals(totals[q, :n], ot), (q, k)
    return docs, totals, n_out


BOOSTS = [-2.5, 3.0, -1e308, -1e308, np.inf, 1e-300, -0.0]


def check_multi(fx, ks, cols, slot_counts=(8, 16)):
    """multi-field top_docs_batch (k_sig_multi TMAX 8 / 16) with negative and -0.0 per-op coefficients, negative and inf
    rule boosts (slot_boost): factors of 0 (two -1e308 downranks sum to inf), inf and tiny make -0.0, +-inf and computed NaN
    totals; against the oracle"""
    oseg = fx["oseg"]
    numeric = [("HostCentrality", 0, 1.0), ("PageCentrality", 1, 1.0)]
    seen = dict(nan=0, negzero=0, neg=0)
    for coefficients in ({"Bm25Title": -0.0, "Bm25CleanBody": -1.0, "HostCentrality": -2.0}, {"TitleCoverage": -0.5, "PageCentrality": 0.0}):
        comp = _multi(fx, cols, coefficients, numeric)
        for ns in slot_counts:
            for k in ks:
                sf = np.full((4, ns), 0xFF, np.uint8); st = np.full((4, ns), NO_TERM, np.uint32)
                boost = np.zeros((4, ns), np.float64)
                for q in range(4):
                    sf[q, :2] = [0, 1]; st[q, :2] = [R.term_of_df(fx, 2 * k + 1), R.term_of_df(fx, k + (q & 1))]
                    if q == 3:   # k candidates, all in the top k: NaN totals (ranked last) are returned too
                        st[q, :2] = R.term_of_df(fx, k)
                    nb = min(ns - 2, 2 + q)          # rule slots: docsets of other terms, with the boosts above
                    for j in range(nb):
                        sf[q, 2 + j] = 0x80 | (j & 1); st[q, 2 + j] = R.term_of_df(fx, [k, 2 * k, k + 1, 2 * k + 1][j % 4])
                        boost[q, 2 + j] = BOOSTS[(q + j) % len(BOOSTS)] if q != 3 else -1e308
                docs, totals, n_out = multi_vs_oracle(comp, oseg, cols, sf, st, k, boost)
                for q in range(4):
                    t = totals[q, :n_out[q]]
                    seen["nan"] += int(np.isnan(t).sum()); seen["neg"] += int((t < 0).sum())
                    seen["negzero"] += int((R.bits(t) == 0x8000000000000000).sum())
    assert all(v > 0 for v in seen.values()), seen


def landing_index(seed, max_doc, n_q, m):
    """A field whose query (Q, P) makes k_sig_multi's candidate count land on the buffer's size: Q is tie-scored with
    n_q postings, P has one posting.  Round 1 takes Q's first m docs and P's doc (bound = P's doc), round 2 the rest of
    Q's first block, then 128 per round; so the running count is m + 1, 129, 129 + 128 j and one round makes it cap + 1
    exactly.  With P's doc inside Q (term P2) it is 128 + 128 j, which lands on cap.  A numeric column rising with the doc
    makes every later candidate the better one, so a candidate lost past the buffer's end changes the top-k.  The kernel
    exposes no per-round count: that its rounds land where this arithmetic says rests on the mutation check of DESIGN §7
    (`have + R > P.cap + 32` fails test_multi_field_buffer_lands_on_cap), not on an assertion here."""
    rng = np.random.default_rng(seed)
    q = np.sort(rng.choice(np.arange(0, max_doc, 2), n_q, replace=False)).astype(np.uint32)
    p1 = np.array([q[m - 1] + 1], np.uint32)       # odd: not in Q, between Q's m-th and (m+1)-th doc
    p2 = np.array([q[m - 1]], np.uint32)
    assert q[m - 1] < p1[0] < q[m]
    docs = [q, p1, p2]
    fx = dict(docs=docs, tfs=[np.ones(d.size, np.uint32) for d in docs], ids=np.full(max_doc, R.FIELDNORM_ID, np.uint8))
    fx["oseg"], fx["seg"] = T.build(fx["docs"], fx["tfs"], None, fieldnorm_ids=fx["ids"])
    return fx


def check_landing(max_doc=200_000, k=1024, ns=8):
    """k_sig_multi at have + R == cap + 1 and == cap (see landing_index); every candidate pushed is the best so far"""
    cap = R.next_pow2(k + ns * 128, 1024)
    n_q = cap + 256
    fx = landing_index(5, max_doc, n_q, 100)
    col = np.arange(max_doc, dtype=np.float64)
    comp = MultiFieldSignalComputer({"Title": fx["seg"]}, {"Bm25Title"}, SignalTable([col]), [("HostCentrality", 0, 1.0)])
    sf = np.full((2, ns), 0xFF, np.uint8); st = np.full((2, ns), NO_TERM, np.uint32)
    sf[:, :2] = 0; st[0, :2] = [0, 1]; st[1, :2] = [0, 2]
    assert (cap - 128) % 128 == 0   # 129 + 128 j reaches cap + 1 (and 128 + 128 j reaches cap) at j = cap / 128 - 1
    docs, totals, n = comp.top_docs_batch(sf, st, k)
    for q in range(2):
        cand = np.union1d(fx["docs"][0], fx["docs"][1 + q])
        want = cand[::-1][:k]
        assert int(n[q]) == k and np.array_equal(docs[q, :k], want), q
    multi_vs_oracle(comp, fx["oseg"], [col], sf, st, k)


def make_split(seed, max_doc, heavy_dfs):
    fx = R.split_index(seed, max_doc, heavy_dfs)
    fx["oseg"], fx["seg"] = T.build(fx["docs"], fx["tfs"], None, fieldnorm_ids=fx["ids"])
    return fx


def check_split(fx, cases, sig=True):
    """`cases` = [(heavy index, k, expected W)].  The batch (heavy + its boundary term, 40 light queries) cuts the heavy query
    into W ranges (plan_items restated); OR (k_or3 + k_merge_topk<0>), the signal combine (k_or3 MODE 2 + k_merge_topk<2>)
    and AND of the heavy term alone (k_topk_warp<AND>) give the same results as the query alone (W = 1) and as the oracle.
    The top of (heavy OR boundary) is the boundary docs max_doc*c/W - 1, max_doc*c/W, max_doc*c/W + 1, all of one score."""
    seg, oseg = fx["seg"], fx["oseg"]
    for h, k, W in cases:
        rows = R.split_batch(fx, h)
        assert R.plan_w(R.work_of(fx, rows), k)[0] == W, (h, k, R.plan_w(R.work_of(fx, rows), k)[0], W)
        assert R.plan_w(R.work_of(fx, rows[:1]), k)[0] == 1
        bounds = R.range_bounds(fx["max_doc"], W)
        assert all(b - 1 in fx["edge"] and b in fx["edge"] and b + 1 in fx["edge"] for b in bounds)
        for mode, omode in ((MODE_OR, 2), (MODE_AND, 2)):
            r = rows if mode == MODE_OR else np.array([[fx["heavy"][h], NO_TERM]] + [[t, NO_TERM] for t in fx["light"]], np.uint32)
            gd, gs, gn = TopDocs.with_limit(k).search_batch(seg, r, mode)
            ad, as_, an = TopDocs.with_limit(k).search_batch(seg, r[:1], mode)
            m = int(gn[0])
            assert m == int(an[0]) and np.array_equal(gd[0, :m], ad[0, :m]) and np.array_equal(gs[0, :m], as_[0, :m]), (mode, h, k)
            _compare(gd[:1], gs[:1], gn[:1], r[:1], oseg, seg, omode, k, ("split", mode))
            if mode == MODE_OR:
                e = fx["edge"][:k]
                assert np.array_equal(gd[0, :e.size], e) and np.unique(gs[0, :e.size]).size == 1
        if sig:
            cols = [np.where(np.isin(np.arange(fx["max_doc"]), fx["edge"]), -0.0, 0.0), R.special_columns(fx["max_doc"], 3)[1]]
            for coeff_text, coeffs in ((0.005, [1.0, 0.0]), (-0.005, [1.0, 1.0])):
                comp = SignalComputer(seg, SignalTable(cols), coeffs, coeff_text=coeff_text)
                gd, gt, gn = comp.top_docs_batch(rows, k)
                ad, at, an = comp.top_docs_batch(rows[:1], k)
                m = int(gn[0])
                assert m == int(an[0]) and np.array_equal(gd[0, :m], ad[0, :m]) and R.same_totals(gt[0, :m], at[0, :m])
                qq = rows[0]
                w = np.array([bm25.StractBm25Weight.for_one_term(int(seg.doc_freq[t]), seg.max_doc, seg.average_fieldnorm).weight for t in qq], np.float32)
                od, ot, _ = oseg.signal_topk(qq, w, np.tile(bm25.compute_tf_cache(seg.average_fieldnorm), (2, 1)), 1.2, coeff_text, cols, coeffs, k)
                assert m == od.size and np.array_equal(gd[0, :m], od) and R.same_totals(gt[0, :m], ot), (h, k, coeff_text)


# ------------------------------------------------------------------ tests -------------------------------------------------
@pytest.fixture(scope="module")
def tie():
    return make_tie(61, GPU_MAX_DOC, R.boundary_ks())


def test_boundary_k_bm25(tie):
    check_boundary_k(tie, R.boundary_ks())


def test_k_out_of_range_refused(tie):
    check_k_refused(tie)


def test_boundary_k_signal_combine_special_totals(tie):
    check_signals(tie, R.boundary_ks(), R.special_columns(GPU_MAX_DOC, 7))


def test_boundary_k_multi_field_special_totals(tie):
    check_multi(tie, [1, 33, 1024, 1025, 2048, 2049, 3072, 3073, 4096], R.special_columns(GPU_MAX_DOC, 8))


def test_multi_field_buffer_lands_on_cap():
    for k, ns in ((1024, 8), (1, 8), (2048, 16)):
        check_landing(k=k, ns=ns)


def test_split_batches():
    """W = 16 at k = 1 and 1024, W = 15 at k = 1025, W = 4 at k = 4096, W = 2; prints runtime and peak host RSS"""
    t0 = time.time()
    fx = make_split(71, SPLIT_MAX_DOC, [W16_DF, W2_DF])
    check_split(fx, [(0, 1, 16), (0, 1024, 16), (0, 1025, 15), (0, 4096, 4), (1, 10, 2), (1, 4096, 2)])
    print(f"split batches: {time.time() - t0:.1f} s; peak host RSS {resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20:.2f} GB")


def test_h100_nan_bits():
    """Records the NaN bits the GPU's f64 units write for 0 * inf, inf - inf and a NaN operand (printed), and checks that
    the top-k hands every NaN total over as 0xFFF8000000000000 whatever those bits are"""
    import torch
    z = torch.tensor([0.0, np.inf, R.NAN_P, R.NAN_N], dtype=torch.float64, device="cuda")
    prod = (z[0:1] * z[1:2]).cpu().numpy(); diff = (z[1:2] - z[1:2]).cpu().numpy(); prop = (z[2:] * 2.0).cpu().numpy()
    print("H100 f64 NaN bits: 0*inf %016x, inf-inf %016x, +NaN*2 %016x, -NaN*2 %016x" %
          (R.bits(prod)[0], R.bits(diff)[0], R.bits(prop)[0], R.bits(prop)[1]))
    fx = make_tie(62, 20_000, [1, 32])
    col = np.full(20_000, np.inf)
    for coeff_text, coeffs, cols in ((0.0, [0.0], [col]), (1.0, [1.0, -1.0], [col, col])):
        comp = SignalComputer(fx["seg"], SignalTable(cols), coeffs, coeff_text=coeff_text)
        d, t, n = comp.top_docs_batch(np.array([[R.term_of_df(fx, 32)]], np.uint32), 32)
        assert n[0] == 32 and np.all(R.bits(t[0, :32]) == 0xFFF8000000000000) and np.array_equal(d[0, :32], fx["docs"][R.term_of_df(fx, 32)][:32])


# ------------------------------------------------------------------ optic=, plan=, webpages, phrases, segments -------------
def _pairs(fx):
    return {"Title": (fx["oseg"], fx["seg"]), "CleanBody": (fx["oseg"], fx["seg"])}


def _two_field_slots(fx, k, nq, ns=8):
    sf = np.full((nq, ns), 0xFF, np.uint8); st = np.full((nq, ns), NO_TERM, np.uint32)
    for q in range(nq):
        sf[q, :2] = [0, 1]; st[q, :2] = [R.term_of_df(fx, 2 * k + 1), R.term_of_df(fx, k + (q & 1))]
    return sf, st


def check_optic(fx, ks, cols):
    """top_docs_batch(optic=) (k_sig_multi<OPTIC>): rule docsets with the boosts that give factors 0, inf and NaN, exclude
    and require, against the multi-field oracle's totals filtered and boosted by pattern_oracle.optic_topk"""
    import test_optic_gpu as TO
    from stract_b200.bm25 import Docset, OpticTables
    comp = _multi(fx, cols, {"Bm25CleanBody": -1.0, "HostCentrality": -2.0}, [("HostCentrality", 0, 1.0), ("PageCentrality", 1, 1.0)])
    seen = dict(nan=0, negzero=0, neg=0)
    for k in ks:
        terms = [R.term_of_df(fx, d) for d in (k, 2 * k, k + 1, 2 * k + 1)]
        docsets = [Docset.from_postings(fx["seg"], t) for t in terms]
        sets = [set(fx["docs"][t].tolist()) for t in terms]
        nq = 6
        sf, st = _two_field_slots(fx, k, nq)
        rules = [[(j % 4, BOOSTS[(q + j) % len(BOOSTS)] if q != 5 else -1e308) for j in range(q)] for q in range(nq)]
        exclude = [None, None, 3, None, None, None]
        require = [None, None, None, 2, None, None]
        tables = OpticTables(docsets, rules, exclude, require)
        docs, totals, n_out = comp.top_docs_batch(sf, st, k, optic=tables)
        want = TO.oracle_recall(comp, _pairs(fx), cols, sf, st, k, tables, sets)
        for q in range(nq):
            n = int(n_out[q])
            assert n == len(want[q]), (k, q, n, len(want[q]))
            assert np.array_equal(docs[q, :n], np.array([d for _, d in want[q]], np.uint32)), (k, q)
            assert R.same_totals(totals[q, :n], [t for t, _ in want[q]]), (k, q)
            t = totals[q, :n]
            seen["nan"] += int(np.isnan(t).sum()); seen["neg"] += int((t < 0).sum())
            seen["negzero"] += int((R.bits(t) == 0x8000000000000000).sum())
        for d in docsets:
            d.close()
    assert all(v > 0 for v in seen.values()), seen


def check_plan(fx, ks, cols):
    """top_docs_batch(plan=) (k_plan_recall, rcap = k + 32 rounded up to a power of two): Must / Should / MustNot TERM
    programs whose docsets hold more than k documents, against the multi-field oracle's totals over the plan's docs"""
    import plan_oracle as PLO
    import pattern_oracle as PO
    import test_optic_gpu as TO
    import test_recall_plan_gpu as TP
    from stract_b200.bm25 import PLAN_BOOL, PLAN_TERM, OpticTables, RecallPlan
    M, S, N = TP.M, TP.S, TP.N
    comp = _multi(fx, cols, {"Bm25CleanBody": -1.0, "HostCentrality": -2.0}, [("HostCentrality", 0, 1.0), ("PageCentrality", 1, 1.0)])
    max_doc = fx["seg"].max_doc
    post = [fx["docs"], fx["docs"]]
    for k in ks:
        a, b, c = R.term_of_df(fx, 2 * k + 1), R.term_of_df(fx, 2 * k), R.term_of_df(fx, k + 1)
        progs = [[(PLAN_TERM, M, 0, 0, a), (PLAN_BOOL, M, 1, 0, 0)],
                 [(PLAN_TERM, S, 0, 0, a), (PLAN_TERM, S, 0, 1, b), (PLAN_BOOL, M, 2, 0, 0)],
                 [(PLAN_TERM, M, 0, 1, a), (PLAN_TERM, N, 0, 0, c), (PLAN_BOOL, M, 2, 0, 0)]]
        plan = RecallPlan([fx["seg"], fx["seg"]], progs)
        want_sets = [PLO.program_docs(p, post) for p in progs]
        assert len(want_sets[0]) > k
        sf, st = _two_field_slots(fx, k, len(progs))
        docs, totals, n_out = comp.top_docs_batch(sf, st, k, plan=plan)
        union = TO.oracle_recall(comp, _pairs(fx), cols, sf, st, max_doc, OpticTables([], [[] for _ in progs]), [])
        for q in range(len(progs)):
            tot = {d: t for t, d in union[q]}
            want = PO.optic_topk([(d, tot[d] if d in tot else TP.zero_text_total(comp, cols, d)) for d in want_sets[q]], k)
            n = int(n_out[q])
            assert n == len(want), (k, q, n, len(want))
            assert np.array_equal(docs[q, :n], np.array([d for _, d in want], np.uint32)), (k, q)
            assert R.same_totals(totals[q, :n], [t for t, _ in want]), (k, q)


def check_webpages(fx, ks, cols):
    """ranking_webpages over each query's top-k: sum(coeff * score) * boost, in op order, equals the top-k total bit for bit
    (any NaN equal to any NaN), negative and -0.0 totals included"""
    comp = _multi(fx, cols, {"Bm25Title": -0.0, "Bm25CleanBody": -1.0, "HostCentrality": -2.0},
                  [("HostCentrality", 0, 1.0), ("PageCentrality", 1, 1.0)])
    coeffs = [comp.coefficient(name, coef) for name, _kind, _f, _c, _col, coef in comp.order.entries]
    seen = dict(negzero=0, neg=0)
    for k in ks:
        nq, ns = 4, 8
        sf, st = _two_field_slots(fx, k, nq, ns)
        boost = np.zeros((nq, ns))
        st[1, :2] = st[3, :2] = R.term_of_df(fx, k)   # k candidates: the negative ones (factor ~1e-308, 0) reach the top k
        for q in range(nq):
            for j in range(2 + q):
                sf[q, 2 + j] = 0x80 | (j & 1); st[q, 2 + j] = R.term_of_df(fx, [k, 2 * k][j & 1])
                boost[q, 2 + j] = -1e308 if q == 3 else BOOSTS[(q + j) % len(BOOSTS)]
        td, tt, tn = comp.top_docs_batch(sf, st, k, slot_boost=boost)
        wp = comp.ranking_webpages(sf, st, td, tn, distance_fields=("-", "-"), slot_boost=boost)   # no min_slop: no positions
        for q in range(nq):
            for i in range(int(tn[q])):
                t = np.float64(0.0)
                with np.errstate(over="ignore", invalid="ignore"):   # inf and NaN totals are the point here
                    for c, s in zip(coeffs, wp.scores[q, i]):
                        t = t + np.float64(c) * np.float64(s)
                    t = t * np.float64(wp.boosts[q, i])
                assert R.same_totals([t], [tt[q, i]]), (k, q, i, t, tt[q, i])
            x = tt[q, :tn[q]]
            seen["neg"] += int((x < 0).sum()); seen["negzero"] += int((R.bits(x) == 0x8000000000000000).sum())
    assert all(v > 0 for v in seen.values()), seen


def _cut(fx, cuts, cols):
    """the tie index cut into segments at `cuts` (device SegmentReaders + their slices of `cols`); term ords per segment"""
    from stract_b200.bm25 import SegmentReader
    segs, ords = [], []
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        sd, present = [], []
        for d in fx["docs"]:
            m = (d >= lo) & (d < hi)
            present.append(len(sd) if m.any() else NO_TERM)
            if m.any():
                sd.append(d[m] - lo)
        data, infos = bm25.encode_postings(sd, [np.ones(x.size, np.uint32) for x in sd], fx["ids"][lo:hi], 1.0)
        segs.append((SegmentReader(data, infos, fx["ids"][lo:hi], total_num_tokens=T.total_num_tokens(fx["ids"][lo:hi])),
                     [c[lo:hi] for c in cols]))
        ords.append(present)
    return segs, ords


def check_segments(fx, ks, cols):
    """Searcher (BM25) and SignalSearcher over the tie index cut into three segments, with the cuts at documents of the
    queried terms, so equal scores and equal totals (NaN, +-inf, negative, tied) lie on both sides of a segment boundary:
    the merged lists equal one segment holding everything (the oracle), with each doc's global id"""
    from stract_b200.bm25 import Searcher, SignalSearcher
    max_doc = fx["seg"].max_doc
    for k in ks:
        a = fx["docs"][R.term_of_df(fx, 2 * k + 1)]
        cuts = [0, int(a[a.size // 3]), int(a[2 * a.size // 3]), max_doc]
        segs, ords = _cut(fx, cuts, cols)
        rows = np.array([[R.term_of_df(fx, 2 * k + 1), R.term_of_df(fx, k)], [R.term_of_df(fx, 2 * k + 1), NO_TERM]], np.uint32)
        per_seg = [np.array([[o[t] if t != NO_TERM else NO_TERM for t in r] for r in rows], np.uint32) for o in ords]
        base = np.array(cuts[:-1], np.uint32)
        sg, dd, sc, n = Searcher([s for s, _ in segs]).search_batch(TopDocs.with_limit(k), per_seg, MODE_OR, n_clauses=[2, 1])
        for q in range(rows.shape[0]):
            qq = np.array([x for x in rows[q] if x != NO_TERM], np.uint32)
            od, os_, _ = fx["oseg"].topk(qq, *T.weights_for(fx["seg"], qq), 2, k)
            m = int(n[q])
            assert m == od.size and np.array_equal(dd[q, :m] + base[sg[q, :m]], od), (k, q)
            assert np.array_equal(sc[q, :m], os_), (k, q)
        for coeff_text, coeffs in COEFFS:
            comps = [SignalComputer(s, SignalTable(c), coeffs, coeff_text=coeff_text) for s, c in segs]
            searcher = SignalSearcher(comps)
            sg, dd, tot, n = searcher.top_docs_batch(per_seg, k)
            cache = bm25.compute_tf_cache(searcher.average_fieldnorm)
            for q in range(rows.shape[0]):
                qq = np.array([x for x in rows[q] if x != NO_TERM], np.uint32)
                w = np.array([bm25.StractBm25Weight.for_one_term(int(fx["seg"].doc_freq[t]), max_doc, searcher.average_fieldnorm).weight
                              for t in qq], np.float32)
                od, ot, _ = fx["oseg"].signal_topk(qq, w, np.tile(cache, (qq.size, 1)), 1.2, coeff_text, cols, coeffs, k)
                m = int(n[q])
                assert m == od.size and np.array_equal(dd[q, :m] + base[sg[q, :m]], od), (k, coeff_text, q)
                assert R.same_totals(tot[q, :m], ot), (k, coeff_text, q)


def check_phrases_k(ks, nq):
    """search_phrase_batch at the boundary k values over the positional range fixture, against the native phrase oracle"""
    import test_postings_range_paths_gpu as P
    fx = P.make(61, P.MEDIUM)
    assert P.check_phrases(fx, np.random.default_rng(9), nq, slops=(0, 3), ks=ks, python_rows=0) > 0
    fx["seg"].close()


def test_boundary_k_optic(tie):
    check_optic(tie, [1, 33, 1024, 1025, 4096], R.special_columns(GPU_MAX_DOC, 8))


def test_boundary_k_plan_recall(tie):
    check_plan(tie, [1, 992, 993, 4064, 4065, 4096], R.special_columns(GPU_MAX_DOC, 8))


def test_boundary_k_ranking_webpages(tie):
    check_webpages(tie, [1, 33, 1025, 4096], R.special_columns(GPU_MAX_DOC, 8))


def test_boundary_k_segments(tie):
    check_segments(tie, [1, 32, 33, 1024, 1025, 4096], R.special_columns(GPU_MAX_DOC, 7))


def test_boundary_k_phrases():
    check_phrases_k([1, 31, 32, 33, 127, 128, 129, 1023, 1024, 1025, 4095, 4096], 12)
