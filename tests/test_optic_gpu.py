"""Optic pattern rules as device docsets (bm25_pattern.cuh) and their use in the multi-field recall stage, against the plain
oracle of tests/pattern_oracle.py: docsets bit-exact as document lists, recall-stage docs and f64 totals bit-exact.  The
check_* functions also run, reduced, on the CPU SIMT emulator (test_optic_emulated.py)."""
import numpy as np
import pytest

import oracle
import pattern_oracle as PO
import phrase_fixtures as F
from stract_b200 import bm25
from stract_b200._lib import Sb200Error
from stract_b200.bm25 import (ABSENT_TERM, NO_TERM, PART_ANCHOR, PART_TERM, PART_WILDCARD, Docset, MultiFieldSignalComputer,
                              OpticTables, SignalTable, pattern_docsets)

pytestmark = pytest.mark.gpu

KIND = {"T": PART_TERM, "*": PART_WILDCARD, "|": PART_ANCHOR}


def doc_tokens(index):
    """The token stream of every document, rebuilt from the index's positions."""
    n = index["fieldnorm_ids"].size
    toks = [dict() for _ in range(n)]
    for t, term in enumerate(index["terms"]):
        for d, pos in zip(term["docs"], term["positions"]):
            for p in pos:
                toks[int(d)][int(p)] = t
    return [[m[i] for i in range(len(m))] for m in toks]


def random_patterns(rng, n_vocab, n):
    """1-8 terms with wildcards, anchors at the start / end / middle, duplicate and absent terms, plus the term-free forms."""
    out = [([], []), (["*"], []), (["|"], []), (["|", "|"], []), (["|", "*", "|"], []), (["T"], [3]), (["T"], [None]),
           (["|", "T"], [0]), (["T", "|"], [1]), (["T", "T"], [0, 1]), (["|", "T", "T", "|"], [0, 1]), (["T", "T"], [2, 2]),
           (["*", "T"], [1]), (["T", "*"], [0]), (["T", "|", "T"], [0, 0])]
    p = 1.0 / np.arange(1, n_vocab + 3) ** 0.5
    p /= p.sum()
    while len(out) < n:
        nt = int(rng.integers(1, 9))
        terms = [int(x) for x in rng.choice(n_vocab + 2, nt, p=p)]
        if nt > 1 and rng.random() < 0.3:
            terms[1] = terms[0]
        if rng.random() < 0.05:
            terms[-1] = None
        parts = []
        for i in range(nt):
            if rng.random() < 0.25:
                parts.append("*")
            if 0 < i and rng.random() < 0.1:
                parts.append("|")
            parts.append("T")
        if rng.random() < 0.4:
            parts.insert(0, "|")
        if rng.random() < 0.4:
            parts.append("|" if rng.random() < 0.7 else "*")
        out.append((parts, terms))
    return out


def to_rows(pats):
    return [([KIND[x] for x in parts], [ABSENT_TERM if t is None else t for t in terms]) for parts, terms in pats]


def check_random_patterns(n_docs=3001, n_pat=160, seed=7):
    index, rng = F.random_index(seed, n_docs)
    toks = doc_tokens(index)
    counts = np.array([len(t) for t in toks], np.uint64)
    counts[rng.choice(np.arange(1, n_docs), 20, replace=False)] = 0       # missing values (passed as 0)
    seg = F.make_segment(index)
    seg.attach_token_counts(counts)
    n_vocab = len(index["terms"]) - 2
    pats = random_patterns(rng, n_vocab, n_pat)
    pats.append((["T", "T"], [0, 1]))                                     # doc 0: tf 1500 each, the global-scratch pass
    pats.append((["|", "T", "*", "T", "|"], [0, 1]))
    got, st = pattern_docsets(seg, to_rows(pats), return_stats=True)
    assert st["candidates"] > 0 and st["positions_decoded"] > 0
    for (parts, terms), d in zip(pats, got):
        want = PO.pattern_docs(toks, parts, terms, [int(c) for c in counts])
        assert np.array_equal(d.docs(), np.array(want, np.uint32)), (parts, terms, d.count(), len(want))
        assert d.count() == len(want)
    # AND / OR combines against set algebra
    a, b, c = got[7], got[9], got[1]
    for op, fn in (("and", lambda x, y: x & y), ("or", lambda x, y: x | y)):
        want = set(a.docs().tolist())
        for x in (b, c):
            want = fn(want, set(x.docs().tolist()))
        assert np.array_equal(Docset.combine(op, [a, b, c]).docs(), np.array(sorted(want), np.uint32))
    # one posting list
    for t in (0, n_vocab, n_vocab + 1):
        assert np.array_equal(Docset.from_postings(seg, t).docs(), index["terms"][t]["docs"])
    assert Docset.from_postings(seg, ABSENT_TERM).count() == 0
    # the capped read returns the first documents
    assert np.array_equal(got[1].docs(cap=5), np.arange(5, dtype=np.uint32))
    return seg


def check_error_paths(n_docs=700):
    index, rng = F.random_index(3, n_docs)
    seg = F.make_segment(index)
    with pytest.raises(Sb200Error) as e:                                    # anchored / empty-field without token counts
        pattern_docsets(seg, to_rows([(["|", "T"], [0])]))
    assert e.value.code == -1   # SB200_EINVAL
    with pytest.raises(Sb200Error):
        pattern_docsets(seg, to_rows([(["|"], [])]))
    pattern_docsets(seg, to_rows([(["T", "T"], [0, 1])]))                # unanchored positional patterns need none
    with pytest.raises(ValueError):                                        # the host mirror's term limit
        pattern_docsets(seg, to_rows([(["T"] * 9, [0] * 9)]))
    from stract_b200 import _lib_bm25 as B
    import ctypes as C
    parts = np.full((1, 9), PART_TERM, np.uint8); ords = np.zeros((1, 9), np.uint32)
    pb = B.PatternBatch(); pb.n_patterns, pb.n_parts, pb.parts, pb.n_terms, pb.term_ords = 1, 9, parts.ctypes.data, 9, ords.ctypes.data
    hs = (C.c_void_p * 1)()
    assert seg._L.sb200_pattern_docsets(seg._h, C.byref(pb), C.cast(hs, C.c_void_p), None) == -4   # SB200_ERANGE
    other, _ = F.random_index(4, n_docs + 1)
    seg2 = F.make_segment(other)
    with pytest.raises(Sb200Error):                                         # max_doc mismatch
        Docset.combine("or", [Docset.from_postings(seg, 0), Docset.from_postings(seg2, 0)])


# ---------------------------------------------------------------------------------------------------- recall stage --------
FIELDS = ["Title", "CleanBody", "Url"]
ENABLED = {"Bm25F", "Bm25Title", "TitleCoverage", "Bm25CleanBody", "CleanBodyCoverage", "IdfSumUrl"}


def make_fields(seed, max_doc):
    import test_bm25_gpu as T
    dfs = {"Title": [40, 300, 129, 2500, 7], "CleanBody": [900, 6000, 128, 15000, 3000, 1], "Url": [20, 500, 4000]}
    mean = {"Title": 2.0, "CleanBody": 5.0, "Url": 1.5}
    out = {}
    for i, f in enumerate(FIELDS):
        rng = np.random.default_rng(seed + i)
        lens = np.maximum(1, rng.lognormal(mean[f], 0.7, max_doc)).astype(np.uint32)
        td = [np.sort(rng.choice(max_doc, min(df * max_doc // 30_000 + 1, max_doc), replace=False)).astype(np.uint32) for df in dfs[f]]
        tt = [np.minimum(rng.geometric(0.6, x.size), 255).astype(np.uint32) for x in td]
        oseg, seg = T.build(td, tt, lens)
        out[f] = (oseg, seg, td, lens)
    return out


def oracle_recall(comp, pairs, cols, sf, st, k, tables, sets):
    """The multi-field oracle's every-candidate totals (k = max_doc), then the optic filters and boosts (pattern_oracle)."""
    names = comp.names
    max_doc = comp.readers[0].max_doc
    osegs = [pairs[n][0] for n in names]
    coefs = [np.float32(comp.field_coefficient(n)) for n in names]
    ops = [(kind, names.index(field) if field is not None else 0, chain, col, comp.coefficient(name, coef))
           for name, kind, field, chain, col, coef in comp.order.entries]
    out = []
    for q in range(sf.shape[0]):
        od, ot = oracle.multi_signal_topk(osegs, comp.last_inputs["caches"], [1.2] * len(names), coefs, sf[q], st[q],
                                          comp.last_inputs["idf"][q], comp.last_inputs["idf_f"][q], ops, cols, max_doc)
        rules = [(sets[i], b) for i, b in tables.rules[q]]
        ex = None if tables.exclude[q] is None else sets[tables.exclude[q]]
        rq = None if tables.require[q] is None else sets[tables.require[q]]
        out.append(PO.optic_topk(zip(od, ot), k, rules, ex, rq))
    return out


def check_optic_batch(max_doc=30_000, nq=24, k=100, seed=21):
    pairs = make_fields(seed, max_doc)
    rng = np.random.default_rng(seed)
    cols = [rng.random(max_doc)]
    comp = MultiFieldSignalComputer({n: pairs[n][1] for n in FIELDS}, ENABLED, SignalTable(cols), [("HostCentrality", 0, 1.0)])
    # rule docsets: posting lists of every field, their AND / OR, All and EmptyField (token counts with zeros)
    title = pairs["Title"][1]
    counts = pairs["Title"][3].astype(np.uint64)
    counts[rng.choice(max_doc, max_doc // 50, replace=False)] = 0
    title.attach_token_counts(counts)
    docsets, sets = [], []
    for f in FIELDS:
        for t, docs in enumerate(pairs[f][2]):
            docsets.append(Docset.from_postings(pairs[f][1], t)); sets.append(set(docs.tolist()))
    n_post = len(docsets)
    for op, fn in (("and", set.intersection), ("or", set.union)):
        for _ in range(4):
            idx = [int(x) for x in rng.choice(n_post, 3, replace=False)]
            docsets.append(Docset.combine(op, [docsets[i] for i in idx])); sets.append(fn(*[sets[i] for i in idx]))
    alld, empty = pattern_docsets(title, to_rows([(["*"], []), (["|", "|"], [])]))
    docsets += [alld, empty]; sets += [set(range(max_doc)), set(np.flatnonzero(counts == 0).tolist())]
    for d, s in zip(docsets, sets):
        assert np.array_equal(d.docs(), np.array(sorted(s), np.uint32))
    nd = len(docsets)
    sf = np.full((nq, 6), 0xFF, np.uint8); st = np.full((nq, 6), NO_TERM, np.uint32)
    rules, exclude, require = [], [], []
    for q in range(nq):
        x = 0
        for fi, name in enumerate(FIELDS):
            for _ in range(int(rng.integers(1, 3))):
                sf[q, x] = fi; st[q, x] = int(rng.integers(0, len(pairs[name][2]))); x += 1
        nr = [0, 1, 8, 64][q % 4]
        rules.append([(int(rng.integers(0, nd)), float(rng.choice([-4.0, -1.0, 0.5, 2.0, 3.0, 100.0]))) for _ in range(nr)])
        exclude.append(None if q % 3 == 0 else int(rng.integers(0, n_post)))
        require.append(None if q % 5 < 2 else int(rng.integers(n_post, nd)))
    tables = OpticTables(docsets, rules, exclude, require)
    docs, totals, n_out = comp.top_docs_batch(sf, st, k, optic=tables)
    want = oracle_recall(comp, pairs, cols, sf, st, k, tables, sets)
    for q in range(nq):
        n = int(n_out[q])
        assert n == len(want[q]), (q, n, len(want[q]))
        assert np.array_equal(docs[q, :n], np.array([d for _, d in want[q]], np.uint32)), q
        assert np.array_equal(totals[q, :n].view(np.uint64), np.array([t for t, _ in want[q]], np.float64).view(np.uint64)), q
    # an empty optic gives the bits of the existing entry point
    d0, t0, n0 = comp.top_docs_batch(sf, st, k)
    d1, t1, n1 = comp.top_docs_batch(sf, st, k, optic=OpticTables([], [[] for _ in range(nq)]))
    assert np.array_equal(n0, n1)
    for q in range(nq):
        n = int(n0[q])
        assert np.array_equal(d0[q, :n], d1[q, :n]) and np.array_equal(t0[q, :n].view(np.uint64), t1[q, :n].view(np.uint64))
    # error paths: rule slots mixed with docset rules, too many rules, a docset of another segment
    sfr = sf.copy(); str_ = st.copy(); sfr[0, 5] = 0x80 | 1; str_[0, 5] = 0
    with pytest.raises(Sb200Error):
        comp.top_docs_batch(sfr, str_, k, slot_boost=np.ones(sf.shape), optic=OpticTables(docsets, [[(0, 1.0)]] + [[] for _ in range(nq - 1)]))
    with pytest.raises(ValueError):
        OpticTables(docsets, [[(0, 1.0)] * 65] + [[] for _ in range(nq - 1)])
    other = make_fields(seed + 9, max_doc + 1)
    with pytest.raises(Sb200Error):
        comp.top_docs_batch(sf, st, k, optic=OpticTables([Docset.from_postings(other["Url"][1], 0)], [[(0, 1.0)] for _ in range(nq)]))


def check_compiled_optic(max_doc=30_000, seed=5):
    """stract_b200.optic: rules, blocked hosts and DiscardNonMatching compiled to tables, the same batch against the oracle."""
    from stract_b200 import optic as O
    pairs = make_fields(seed, max_doc)
    readers = {n: pairs[n][1] for n in FIELDS}
    # a synthetic resolver: raw text "f<i>" is term i of the field (exact lookups on Url only)
    resolve = lambda field, text, exact: [int(text[1:])] if text[1:].isdigit() and int(text[1:]) < len(pairs[field][2]) else [ABSENT_TERM]
    fields = {"Title": readers["Title"], "CleanBody": readers["CleanBody"], "Url": readers["Url"]}
    opt1 = O.Optic([O.Rule([[O.Matching("t0", "Title")], [O.Matching("t1", "Content"), O.Matching("t3", "Content")]], O.Action.boost(3)),
                    O.Rule([[O.Matching("t2", "Url")]], O.Action.downrank(2)),
                    O.Rule([[O.Matching("t1", "Url")]], O.Action.DISCARD),
                    O.Rule([[O.Matching("t1", "Title")]]),                                   # Boost(0): not a boost, in require
                    O.Rule([], O.Action.boost(5))], discard_non_matching=True)
    opt2 = O.Optic([O.Rule([[O.Matching("t4", "Content")]], O.Action.boost(1))])
    tables = O.compile_optics(fields, [[opt1], [opt2], [opt1, opt2], []], resolve)
    assert [len(r) for r in tables.rules] == [2, 1, 3, 0]
    sets = [set(d.docs().tolist()) for d in tables.docsets]
    P = lambda f, t: set(pairs[f][2][t].tolist())
    r0 = P("Title", 0) | (P("CleanBody", 1) & P("CleanBody", 3))
    assert sets[tables.rules[0][0][0]] == r0 and tables.rules[0][0][1] == 3.0 and tables.rules[0][1][1] == -2.0
    assert sets[tables.exclude[0]] == P("Url", 1) and tables.exclude[1] is None
    assert sets[tables.require[0]] == r0 | P("Url", 2) | P("Title", 1) and tables.require[1] is None
    assert sets[tables.require[2]] == sets[tables.require[0]]
    rng = np.random.default_rng(seed)
    cols = [rng.random(max_doc)]
    comp = MultiFieldSignalComputer(readers, ENABLED, SignalTable(cols), [("HostCentrality", 0, 1.0)])
    sf = np.full((4, 4), 0xFF, np.uint8); st = np.full((4, 4), NO_TERM, np.uint32)
    sf[:, :3] = [0, 1, 2]; st[:, :3] = [3, 3, 2]
    docs, totals, n_out = comp.top_docs_batch(sf, st, 200, optic=tables)
    want = oracle_recall(comp, pairs, cols, sf, st, 200, tables, sets)
    for q in range(4):
        n = int(n_out[q])
        assert np.array_equal(docs[q, :n], np.array([d for _, d in want[q]], np.uint32))
        assert np.array_equal(totals[q, :n].view(np.uint64), np.array([t for t, _ in want[q]], np.float64).view(np.uint64))


def test_random_pattern_docsets_bit_exact():
    check_random_patterns()


def test_pattern_error_paths():
    check_error_paths()


def test_optic_recall_batch_bit_exact():
    check_optic_batch()


def test_compiled_optics_bit_exact():
    check_compiled_optic()
