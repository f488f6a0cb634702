"""The recall webpages (sb200_multi_signal_webpages, bm25_webpage.cuh) against tests/webpage_oracle.py: per-op values and scores,
boosts and min_slop bit for bit, the top-k totals rebuilt from them bit for bit, and the recall-stage mirror over both.  The
check_* functions also run, reduced, on the CPU SIMT emulator (test_recall_webpages_emulated.py)."""
import numpy as np
import pytest

import phrase_fixtures as F
import webpage_oracle as WO
from stract_b200 import ranking_pipeline as RP
from stract_b200._lib import Sb200Error
from stract_b200.bm25 import (NO_TERM, PLAN_TERM, Docset, MultiFieldSignalComputer, OpticTables, RecallPlan, SegmentReader, SignalTable,
                              encode_postings)

pytestmark = pytest.mark.gpu
FIELDS = ["Title", "CleanBody", "Url", "TitleBigrams"]      # Title / CleanBody with positions, the other two without
ENABLED = {"Bm25F", "Bm25Title", "TitleCoverage", "Bm25TitleBigrams", "Bm25CleanBody", "CleanBodyCoverage", "IdfSumUrl"}
N_VOCAB = 24


def plain_segment(index):
    """an index as a record-option-1 segment: postings and tfs, no positions"""
    terms, ids = index["terms"], index["fieldnorm_ids"]
    avg = np.float32(np.float32(index["total_num_tokens"]) / np.float32(ids.size))
    tfs = [np.array([len(p) for p in t["positions"]], np.uint32) for t in terms]
    data, infos = encode_postings([t["docs"] for t in terms], tfs, ids, avg)
    return SegmentReader(data, infos, ids, total_num_tokens=index["total_num_tokens"])


def make_fields(seed, n_docs, long_doc):
    """Title and CleanBody from token streams with positions (doc 0 of CleanBody: a tf above the shared-memory buffer, positions
    over many blocks; the vint-only term N_VOCAB + 1); Url and TitleBigrams as fields without positions"""
    out = {}
    for i, (name, ld) in enumerate(zip(FIELDS, (40, long_doc, 20, 30))):
        index, _ = F.random_index(seed + 17 * i, n_docs, N_VOCAB, long_doc=ld)
        seg = F.make_segment(index) if name in ("Title", "CleanBody") else plain_segment(index)
        out[name] = (index, seg)
    return out


def random_slots(rng, nq, rules=False):
    """queries of 1..8 terms: every term a slot in Title and CleanBody, short queries also in Url / TitleBigrams; absent terms
    (NO_TERM) and duplicates; `rules`: a Title rule slot (| 0x80) in some queries"""
    sf = np.full((nq, 16), 0xFF, np.uint8); st = np.full((nq, 16), NO_TERM, np.uint32); sb = np.zeros((nq, 16))
    for q in range(nq):
        n = 1 + q % 8
        terms = [int(rng.integers(0, N_VOCAB + 2)) for _ in range(n)]
        if n > 2 and rng.random() < 0.5:
            terms[-1] = terms[0]                                       # a duplicate term: separate slots
        x = 0
        for f in (0, 1):
            for t in terms:
                sf[q, x] = f; st[q, x] = NO_TERM if rng.random() < 0.08 else t; x += 1
        for f in (2, 3):
            if x + n <= 15 and n <= 3:
                for t in terms:
                    sf[q, x] = f; st[q, x] = t; x += 1
        if rules and x < 16 and q % 3 == 0:
            sf[q, x] = 0x80; st[q, x] = int(rng.integers(0, 6)); sb[q, x] = float(rng.choice([-2.0, 0.5, 3.0]))
    return sf, st, sb


def build(seed, n_docs, long_doc):
    fields = make_fields(seed, n_docs, long_doc)
    rng = np.random.default_rng(seed)
    cols = [rng.random(n_docs)]
    comp = MultiFieldSignalComputer({n: fields[n][1] for n in FIELDS}, ENABLED, SignalTable(cols), [("HostCentrality", 0, 1.0)])
    assert comp.names == FIELDS
    return fields, comp, cols, rng


def oracle_for(comp, fields, cols):
    ops = [(kind, comp.names.index(field) if field is not None else 0, chain, col, comp.coefficient(name, coef))
           for name, kind, field, chain, col, coef in comp.order.entries]
    return WO.Oracle([{"terms": fields[n][0]["terms"], "ids": fields[n][0]["fieldnorm_ids"]} for n in comp.names],
                     comp.last_inputs["caches"], comp.k1, [np.float32(comp.field_coefficient(n)) for n in comp.names], ops, cols)


def doc_set(fields, f, t):
    return set(fields[FIELDS[f]][0]["terms"][t]["docs"].tolist())


def oracle_query(O, fields, comp, sf, st, sb, q, tables):
    text = [(x, int(sf[q, x]), int(st[q, x])) for x in range(sf.shape[1]) if sf[q, x] != 0xFF and not sf[q, x] & 0x80]
    slots = [(f, o) for _, f, o in text]
    idf = [comp.last_inputs["idf"][q][x] for x, _, _ in text]
    idf_f = [comp.last_inputs["idf_f"][q][x] for x, _, _ in text]
    rs = [(doc_set(fields, int(sf[q, x]) & 0x7F, int(st[q, x])), float(sb[q, x])) for x in range(sf.shape[1])
          if sf[q, x] != 0xFF and sf[q, x] & 0x80]
    rules = [] if tables is None else [(tables.sets[i], b) for i, b in tables.rules[q]]
    return lambda d: O.page(d, slots, idf, idf_f, rs, rules, dist=(0, 1))


def bits(x):
    return np.asarray(x, np.float64).view(np.uint64)


def check_webpages(n_docs=6_000, nq=48, k=50, seed=3, long_doc=3_000, optic=False):
    """Documents: each query's top-k from the union (or optic) and plan paths, random documents, documents no slot holds, doc 0
    (tf above the shared buffer), duplicates, all shuffled.  Values, scores, boosts and min_slop bit-equal to the oracle; the
    top-k totals rebuilt as sum(coeff * score) * boost bit-equal to the entry points'."""
    fields, comp, cols, rng = build(seed, n_docs, long_doc)
    sf, st, sb = random_slots(rng, nq, rules=not optic)
    tables = None
    if optic:
        ds = [Docset.from_postings(fields["Title"][1], t) for t in range(8)]
        rules = [[(int(rng.integers(0, 8)), float(rng.choice([-2.0, 0.5, 3.0]))) for _ in range(q % 4)] for q in range(nq)]
        exclude = [None if q % 2 else int(rng.integers(0, 8)) for q in range(nq)]   # not applied to the webpages
        tables = OpticTables(ds, rules, exclude)
        tables.sets = [doc_set(fields, 0, t) for t in range(8)]
    boost = None if optic else sb
    td, tt, tn = comp.top_docs_batch(sf, st, k, slot_boost=boost, optic=tables)
    plan = RecallPlan([fields["CleanBody"][1]], [[(PLAN_TERM, 0, 0, 0, int(st[q, 0]) if st[q, 0] != NO_TERM else 0)] for q in range(nq)])
    pd, pt, pn = comp.top_docs_batch(sf, st, k, slot_boost=boost, optic=tables, plan=plan)
    lists, known = [], []
    for q in range(nq):
        top = td[q, :tn[q]].tolist()
        d = top + pd[q, :pn[q]].tolist() + rng.integers(0, n_docs, 20).tolist() + [0, n_docs - 1] + top[:3]
        rng.shuffle(d)
        lists.append(d)
        known.append({int(a): t for a, t in zip(td[q, :tn[q]], tt[q, :tn[q]])} | {int(a): t for a, t in zip(pd[q, :pn[q]], pt[q, :pn[q]])})
    ndm = max(len(x) for x in lists) + 3
    docs = np.zeros((nq, ndm), np.uint32); n = np.array([len(x) for x in lists], np.uint32)
    for q, x in enumerate(lists):
        docs[q, :len(x)] = x
    wp, stats = comp.ranking_webpages(sf, st, docs, n, slot_boost=boost, optic=tables, return_stats=True)
    assert wp.names == [e[0] for e in comp.order.entries]
    O = oracle_for(comp, fields, cols)
    numeric = [o for o, e in enumerate(comp.order.entries) if e[1] == WO.OP_NUMERIC]
    checked = 0
    for q in range(nq):
        page = oracle_query(O, fields, comp, sf, st, sb, q, tables)
        for i, d in enumerate(lists[q]):
            v, s, b, sl = page(d)
            for o in numeric:
                v[o] = np.nan                                      # a plain SignalTable has no raw columns
            assert np.array_equal(bits(wp.values[q, i]), bits(v)), (q, i, d, wp.values[q, i], v)
            assert np.array_equal(bits(wp.scores[q, i]), bits(s)), (q, i, d, wp.scores[q, i], s)
            assert bits(wp.boosts[q, i]) == bits(b), (q, i, d, wp.boosts[q, i], b)
            assert tuple(int(x) for x in wp.min_slop[q, i]) == sl, (q, i, d, wp.min_slop[q, i], sl)
            if d in known[q]:
                assert bits(O.total(wp.scores[q, i], wp.boosts[q, i])) == bits(known[q][d]), (q, i, d)
                checked += 1
        assert np.all(np.isnan(wp.values[q, len(lists[q]):]))
        assert not wp.scores[q, len(lists[q]):].any() and not wp.min_slop[q, len(lists[q]):].any()
    assert checked > nq
    assert stats["docs"] == int(n.sum()) and stats["docs_with_positions"] > 0 and stats["positions_decoded"] > 0
    return comp, fields, wp, lists, known, cols


def check_recall_stage(n_docs=4_000, nq=16, k=40, seed=5, long_doc=600):
    """recall_stage over the device webpages and over the oracle's gives the same order and bit-equal scores and boosts"""
    fields, comp, cols, rng = build(seed, n_docs, long_doc)
    sf, st, sb = random_slots(rng, nq)
    td, tt, tn = comp.top_docs_batch(sf, st, k, slot_boost=sb)
    wp = comp.ranking_webpages(sf, st, td, tn, slot_boost=sb)
    O = oracle_for(comp, fields, cols)
    coefs = RP.default_coefficients()
    inbound = {d: float(x) for d, x in enumerate(rng.random(n_docs))}
    for q in range(nq):
        m = int(tn[q])
        got = RP.recall_stage(RP.pages_from_webpages(wp, q, td[q], m, tt[q]), coefs, inbound)
        page = oracle_query(O, fields, comp, sf, st, sb, q, None)
        want_pages = []
        for i in range(m):
            v, s, b, sl = page(int(td[q, i]))
            p = RP.Page(int(td[q, i]), {name: (v[o], s[o]) for o, name in enumerate(wp.names)}, tt[q, i], b)
            p.min_slop = sl
            want_pages.append(p)
        want = RP.recall_stage(want_pages, coefs, inbound)
        assert [p.key for p in got] == [p.key for p in want], q
        assert all(bits(a.score) == bits(b.score) and bits(a.boost) == bits(b.boost) for a, b in zip(got, want)), q


def check_error_paths(n_docs=800):
    fields, comp, cols, rng = build(11, n_docs, 100)
    sf, st, sb = random_slots(rng, 4)
    docs = np.zeros((4, 3), np.uint32); n = np.full(4, 3, np.uint32)
    comp.ranking_webpages(sf, st, docs, n)
    bad_doc = docs.copy(); bad_doc[2, 1] = n_docs
    with pytest.raises(Sb200Error):
        comp.ranking_webpages(sf, st, bad_doc, n)                          # doc >= max_doc
    with pytest.raises(Sb200Error):
        comp.ranking_webpages(sf, st, docs, np.array([3, 4, 3, 3], np.uint32))   # n_docs > n_docs_max
    with pytest.raises(Sb200Error):
        comp.ranking_webpages(sf, st, docs, n, distance_fields=("Title", "Url"))   # a distance field without positions
    with pytest.raises(Sb200Error):
        comp.ranking_webpages(sf, st, docs, n, distance_fields=("Title", "Title"))
    rs = sf.copy(); rs[0, 15] = 0x80; rst = st.copy(); rst[0, 15] = 1
    tables = OpticTables([Docset.from_postings(fields["Title"][1], 0)], [[(0, 2.0)], [], [], []])
    with pytest.raises(Sb200Error):                                        # rule slots and docset rules in one query
        comp.ranking_webpages(rs, rst, docs, n, slot_boost=np.ones(rs.shape), optic=tables)
    # unregistered distance fields: every min_slop is u32::MAX
    wp = comp.ranking_webpages(sf, st, docs, n, distance_fields=("Keywords", "Description"))
    assert (wp.min_slop == RP.U32_MAX).all()


def check_hand_positions():
    """hand-made token streams: one term, an absent term, b only before a, equal positions (duplicate terms), a clean pair"""
    a, b, c, x = 0, 1, 2, 3
    toks = [[a, x, b], [b, x, a], [a, b, a, b], [c, c], [x], [a, c, x, x, x, b]]
    from test_recall_plan_gpu import index_from_tokens
    index = index_from_tokens(toks)
    seg = F.make_segment(index)
    comp = MultiFieldSignalComputer({"Title": seg}, {"Bm25Title", "TitleCoverage"})
    rows = [[a], [a, 9], [a, b], [b, a], [a, a], [a, c, b]]
    sf = np.full((len(rows), 4), 0xFF, np.uint8); st = np.full((len(rows), 4), NO_TERM, np.uint32)
    for q, r in enumerate(rows):
        sf[q, :len(r)] = 0; st[q, :len(r)] = [t if t < 4 else NO_TERM for t in r]
    docs = np.tile(np.arange(len(toks), dtype=np.uint32), (len(rows), 1)); n = np.full(len(rows), len(toks), np.uint32)
    wp = comp.ranking_webpages(sf, st, docs, n)
    for q, r in enumerate(rows):
        for d, tk in enumerate(toks):
            lists = [[i for i, y in enumerate(tk) if y == t] if t < 4 else [] for t in r]
            assert int(wp.min_slop[q, d, 0]) == RP.min_slop(lists), (r, tk)
            assert int(wp.min_slop[q, d, 1]) == RP.U32_MAX                 # CleanBody is not a field of this computer
    assert int(wp.min_slop[2, 0, 0]) == 2 and int(wp.min_slop[3, 0, 0]) == RP.U32_MAX and int(wp.min_slop[4, 2, 0]) == 2


def test_webpages_bit_exact():
    check_webpages()


def test_webpages_optic_bit_exact():
    check_webpages(optic=True, seed=8)


def test_webpages_recall_stage():
    check_recall_stage()


def test_webpages_error_paths():
    check_error_paths()


def test_webpages_hand_positions():
    check_hand_positions()
