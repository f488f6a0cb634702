"""The query-plan recall docset (bm25_plan.cuh) and the recall stage over it, against tests/plan_oracle.py and the
multi-field oracle: docsets equal as doc lists, recall docs and f64 totals bit-exact.  The check_* functions also run, reduced,
on the CPU SIMT emulator (test_recall_plan_emulated.py)."""
import numpy as np
import pytest

import phrase_fixtures as F
import plan_oracle as PLO
import pattern_oracle as PO
import test_optic_gpu as TO
from stract_b200 import query_plan as QP
from stract_b200._lib import Sb200Error
from stract_b200.bm25 import (ABSENT_TERM, NO_TERM, PLAN_BOOL, PLAN_EMPTY, PLAN_PHRASE, PLAN_TERM, Docset, MultiFieldSignalComputer,
                              OpticTables, RecallPlan, SignalTable, recall_plan_docs)

pytestmark = pytest.mark.gpu
M, S, N = QP.MUST, QP.SHOULD, QP.MUST_NOT
SEGS = TO.FIELDS + ["UrlForSiteOperator"]          # the last one is not a signal field
SCHEMA = QP.Schema(TO.FIELDS, {"Title", "CleanBody"}, {"Title", "Url"}, set())


def make_index(seed, max_doc):
    import test_bm25_gpu as T
    pairs = TO.make_fields(seed, max_doc)
    rng = np.random.default_rng(seed + 77)
    td = [np.sort(rng.choice(max_doc, min(n, max_doc // 2), replace=False)).astype(np.uint32) for n in (3, 40, 700)]
    oseg, seg = T.build(td, [np.ones(x.size, np.uint32) for x in td], np.ones(max_doc, np.uint32))
    pairs["UrlForSiteOperator"] = (oseg, seg, td, None)
    return pairs


def resolver(pairs):
    def r(field, text):
        if field not in pairs:
            return None
        if not text.startswith("t") or not text[1:].isdigit():
            return []                                   # compounds and other texts have no tokens here
        i = int(text[1:])
        return [i] if i < len(pairs[field][2]) else [ABSENT_TERM]
    return r


def random_queries(rng, n):
    out = []
    for _ in range(n):
        terms = [("simple", f"t{int(rng.integers(0, 7))}") for _ in range(int(rng.integers(1, 7)))]
        if rng.random() < 0.3:
            terms.append(("not", ("simple", f"t{int(rng.integers(0, 4))}")))
        if rng.random() < 0.3:
            terms.append(("site", f"t{int(rng.integers(0, 4))}"))
        if rng.random() < 0.2:
            terms.append(("title", ("simple", f"t{int(rng.integers(0, 5))}")))
        out.append(QP.parse(terms, SCHEMA, safe_search=False))
    return out


HAND = [[(PLAN_BOOL, M, 0, 0, 0)],                                                    # empty Boolean
        [(PLAN_TERM, N, 0, 1, 1), (PLAN_BOOL, M, 1, 0, 0)],                            # a single MustNot
        [(PLAN_TERM, M, 0, 0, 0), (PLAN_TERM, S, 0, 1, 3), (PLAN_BOOL, M, 2, 0, 0)],   # Must + Should: Should ignored
        [(PLAN_EMPTY, S, 0, 0, 0), (PLAN_TERM, S, 0, 3, 2), (PLAN_BOOL, M, 2, 0, 0)],  # kept empty clause, non-signal field
        [(PLAN_TERM, M, 0, 2, ABSENT_TERM)],                                           # absent term
        [(PLAN_TERM, N, 0, 0, 1), (PLAN_TERM, N, 0, 1, 2), (PLAN_BOOL, M, 2, 0, 0)],   # neither Must nor Should
        [(PLAN_TERM, S, 0, 1, 1), (PLAN_TERM, S, 0, 1, 3), (PLAN_TERM, N, 0, 0, 3), (PLAN_BOOL, M, 3, 0, 0)]]


def plans(pairs, rng, nq, order=SEGS):
    qs = random_queries(rng, nq)
    plan = QP.compile_plans(qs, {n: pairs[n][1] for n in order}, resolver(pairs), SCHEMA)
    if order != SEGS:   # the hand-made programs address segments in SEGS order
        return plan
    plan.programs += HAND
    plan.n_queries = len(plan.programs)
    return plan


def want_docs(pairs, plan, order=SEGS):
    post = [pairs[n][2] for n in order]
    return [PLO.program_docs(p, post) for p in plan.programs]


def check_docsets(max_doc=30_000, nq=120, seed=3):
    pairs = make_index(seed, max_doc)
    rng = np.random.default_rng(seed)
    plan = plans(pairs, rng, nq)
    got, st = recall_plan_docs(plan, return_stats=True)
    want = want_docs(pairs, plan)
    for q, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g, np.array(w, np.uint32)), (q, plan.programs[q], g.size, len(w))
    assert st["docs"] == sum(len(w) for w in want) and st["cover"] >= st["docs"]
    return pairs, plan, want, st


def zero_text_total(comp, cols, d):
    t = 0.0
    for name, kind, field, chain, col, coef in comp.order.entries:
        sc = float(cols[col][d]) if kind == 4 else 0.0
        t = float(np.float64(t) + np.float64(comp.coefficient(name, coef)) * np.float64(sc))
    return t


def check_plan_batch(max_doc=30_000, nq=40, k=100, seed=9, optic=True, order=SEGS):
    """order: the plan's segment order; with a non-signal field first the docset stage and the recall run on different
    streams.  Queries whose plans match nothing (absent terms only) close the batch, so a small budget leaves groups whose
    covers are all empty."""
    pairs = make_index(seed, max_doc)
    rng = np.random.default_rng(seed)
    plan = plans(pairs, rng, nq, order)
    si = order.index("Url")
    plan.programs += [[(PLAN_TERM, M, 0, si, ABSENT_TERM)]] * 12 + [[(PLAN_BOOL, M, 0, 0, 0)]] * 4
    plan.n_queries = len(plan.programs)
    nq = plan.n_queries
    cols = [rng.random(max_doc)]
    comp = MultiFieldSignalComputer({n: pairs[n][1] for n in TO.FIELDS}, TO.ENABLED, SignalTable(cols), [("HostCentrality", 0, 1.0)])
    sf = np.full((nq, 6), 0xFF, np.uint8); st = np.full((nq, 6), NO_TERM, np.uint32)
    for q in range(nq):
        x = 0
        for fi, name in enumerate(TO.FIELDS):
            for _ in range(int(rng.integers(1, 3))):
                sf[q, x] = fi; st[q, x] = int(rng.integers(0, len(pairs[name][2]))); x += 1
    docsets = [Docset.from_postings(pairs[f][1], t) for f in TO.FIELDS for t in range(len(pairs[f][2]))]
    sets = [set(pairs[f][2][t].tolist()) for f in TO.FIELDS for t in range(len(pairs[f][2]))]
    rules = [[(int(rng.integers(0, len(docsets))), float(rng.choice([-2.0, 0.5, 3.0]))) for _ in range(q % 3)] for q in range(nq)]
    exclude = [None if q % 2 else int(rng.integers(0, len(docsets))) for q in range(nq)]
    require = [None if q % 3 else int(rng.integers(0, len(docsets))) for q in range(nq)]
    tables = OpticTables(docsets, rules, exclude, require) if optic else OpticTables([], [[] for _ in range(nq)])
    for kk in (k, max_doc):                                             # k above every docset size too
        docs, totals, n_out = comp.top_docs_batch(sf, st, min(kk, 4096), optic=tables if optic else None, plan=plan)
        union = TO.oracle_recall(comp, pairs, cols, sf, st, max_doc, OpticTables([], [[] for _ in range(nq)]), [])
        want_sets = want_docs(pairs, plan, order)
        for q in range(nq):
            tot = {d: t for t, d in union[q]}
            cand = [(d, tot[d] if d in tot else zero_text_total(comp, cols, d)) for d in want_sets[q]]
            rl = [(sets[i], b) for i, b in tables.rules[q]]
            ex = None if tables.exclude[q] is None else sets[tables.exclude[q]]
            rq = None if tables.require[q] is None else sets[tables.require[q]]
            want = PO.optic_topk(cand, min(kk, 4096), rl, ex, rq)
            n = int(n_out[q])
            assert n == len(want), (q, n, len(want))
            assert np.array_equal(docs[q, :n], np.array([d for _, d in want], np.uint32)), q
            assert np.array_equal(totals[q, :n].view(np.uint64), np.array([t for t, _ in want], np.float64).view(np.uint64)), q
    return comp, plan, sf, st


def index_from_tokens(docs):
    """A phrase_fixtures index from explicit token lists (term ids)"""
    from stract_b200.bm25 import fieldnorm_table, fieldnorms_to_ids
    n_vocab = max(max(d) for d in docs if d) + 1
    terms = []
    for t in range(n_vocab):
        ds = [i for i, d in enumerate(docs) if t in d]
        terms.append({"docs": np.array(ds, np.uint32), "positions": [np.flatnonzero(np.array(docs[i]) == t).astype(np.uint32) for i in ds]})
    ids = fieldnorms_to_ids(np.array([max(len(d), 1) for d in docs], np.uint32))
    return {"fieldnorm_ids": ids, "terms": terms, "total_num_tokens": int(fieldnorm_table()[ids].astype(np.uint64).sum())}


def phrase_sets(index, plan):
    return [PLO.phrase_exists_docs(index, [None if t == ABSENT_TERM else t for t in terms], list(range(len(terms))) if offs is None else offs, sl)
            for terms, offs, sl in plan.phrases]


def check_phrase_plans(n_docs=2_000, nq=80, seed=7):
    """PHRASE leaves (phrase_exists, slop 0 and 2, absent terms, duplicate terms, offsets) mixed with TERM leaves under every
    occur, on a field with positions next to one without"""
    index, rng = F.random_index(seed, n_docs, long_doc=600)
    seg = F.make_segment(index)
    pairs = make_index(seed, n_docs)
    other = pairs["Url"][1]                                  # segment 1: a field without positions
    n_vocab = len(index["terms"]) - 2
    rows, offs = F.random_rows(rng, n_vocab, 40, 4)
    phrases = []
    for r in range(rows.shape[0]):
        m = int((rows[r] != NO_TERM).sum())
        phrases.append(([int(x) for x in rows[r, :m]], [int(x) for x in offs[r, :m]], int(rng.choice([0, 0, 2]))))
    progs = []
    for _ in range(nq):
        prog, n = [], int(rng.integers(1, 5))
        for _ in range(n):
            occ = int(rng.choice([M, M, S, S, N]))
            x = rng.random()
            if x < 0.5:
                prog.append((PLAN_PHRASE, occ, 0, 0, int(rng.integers(0, len(phrases)))))
            elif x < 0.8:
                prog.append((PLAN_TERM, occ, 0, 0, int(rng.integers(0, n_vocab + 2))))
            else:
                prog.append((PLAN_TERM, occ, 0, 1, int(rng.integers(0, len(pairs["Url"][2])))))
        prog.append((PLAN_BOOL, M, n, 0, 0))
        progs.append(prog)
    progs.append([(PLAN_PHRASE, M, 0, 0, 0)])                # a lone phrase leaf
    plan = RecallPlan([seg, other], progs, phrases)
    got = recall_plan_docs(plan)
    ps = phrase_sets(index, plan)
    post = [[t["docs"] for t in index["terms"]], pairs["Url"][2]]
    for q, prog in enumerate(progs):
        assert np.array_equal(got[q], np.array(PLO.program_docs(prog, post, ps), np.uint32)), (q, prog)
    # the phrase leaf of a field without positions is rejected
    with pytest.raises(Sb200Error):
        recall_plan_docs(RecallPlan([seg, other], [[(PLAN_PHRASE, M, 0, 1, 0)]], phrases))
    return plan


def check_exists_not_count():
    """"b c x x a b" against "c b a"~2: PhraseScorer::phrase_exists and compute_phrase_count > 0 disagree; the recall
    docset follows phrase_exists (scoring is disabled)"""
    import phrase_oracle as O
    a, b, c, x = 0, 1, 2, 3
    docs = [[b, c, x, x, a, b], [c, b, a], [a, b, c], [x, x]]
    index = index_from_tokens(docs)
    seg = F.make_segment(index)
    plan = RecallPlan([seg], [[(PLAN_PHRASE, M, 0, 0, 0)]], [([c, b, a], [0, 1, 2], 2)])
    got = recall_plan_docs(plan)[0]
    want = PLO.phrase_exists_docs(index, [c, b, a], [0, 1, 2], 2)
    counted = [d for _, d in O.phrase_search(index, [c, b, a], [0, 1, 2], 2, True, 1.0, [1.0] * 256, 4)]
    assert (0 in want) != (0 in counted)                     # the case really separates the two predicates
    assert np.array_equal(got, np.array(want, np.uint32))


def check_error_paths(max_doc=2_000):
    pairs = make_index(5, max_doc)
    segs = [pairs[n][1] for n in SEGS]
    bad = [[(PLAN_TERM, M, 0, 0, 0), (PLAN_TERM, M, 0, 0, 1)],          # two values left
           [(PLAN_BOOL, M, 2, 0, 0)],                                  # stack underflow
           [(PLAN_TERM, M, 0, 9, 0)],                                  # segment index
           [(PLAN_TERM, M, 0, 0, 10_000)],                             # ordinal
           [(PLAN_PHRASE, M, 0, 0, 0)],                                # no phrase table
           [(7, M, 0, 0, 0)], [(PLAN_TERM, 5, 0, 0, 0)], [],
           [(PLAN_EMPTY, M, 0, 0, 0)] * 257]
    for prog in bad:
        with pytest.raises(Sb200Error):
            recall_plan_docs(RecallPlan(segs, [prog]))
    other = make_index(6, max_doc + 1)
    with pytest.raises(Sb200Error):
        recall_plan_docs(RecallPlan([segs[0], other["Url"][1]], [[(PLAN_TERM, M, 0, 1, 0)]]))


def test_plan_docsets_equal_oracle():
    check_docsets()


def test_plan_docsets_multi_group(monkeypatch):
    monkeypatch.setenv("SB200_PLAN_BUDGET_MB", "1")
    *_, st = check_docsets(max_doc=200_000, nq=60, seed=4)
    assert st["groups"] > 1


def test_plan_recall_bit_exact():
    check_plan_batch(optic=False)


def test_plan_recall_optic_bit_exact():
    check_plan_batch(optic=True)


def test_plan_error_paths():
    check_error_paths()


def test_plan_phrase_leaves():
    check_phrase_plans()


def test_plan_phrase_exists_not_count():
    check_exists_not_count()


def test_plan_recall_other_stream_and_empty_groups(monkeypatch):
    monkeypatch.setenv("SB200_PLAN_BUDGET_MB", "1")
    check_plan_batch(optic=False, order=["UrlForSiteOperator"] + TO.FIELDS)


def test_plan_recall_multi_group(monkeypatch):
    monkeypatch.setenv("SB200_PLAN_BUDGET_MB", "1")
    comp, plan, sf, st = check_plan_batch(max_doc=150_000, nq=30, optic=True)
    assert recall_plan_docs(plan, return_stats=True)[1]["groups"] > 1
