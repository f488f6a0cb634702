"""Phrase search and optic pattern docsets over the positions format's full range (fixtures: tests/postings_range.py).
Needs a GPU.

The positional index puts the phrase and pattern kernels (k_phrase_cand, k_phrase_verify, the pattern verify) on one
positions block per delta width 0..32, positions from 2^31 up, 1- to 5-byte VInt deltas, a posting of tf 2^16 + 1 (a
verify pass over global scratch), doc ids spread over a ~2^22-doc space with wide doc deltas up to max_doc - 1, and a
three-term carrying-slop phrase that matches only because `slop_so_far as u32 + abs_diff` wraps in u32.  One term's
positions pass 4 GiB of bit-packed data (huge_positions_term), so a per-block byte offset must not be 32-bit.  Bar: docs,
order and f32 score bits equal to the native and the Python phrase oracle, and pattern docsets equal to the pattern oracle
run on the input positions."""
import resource
import time

import numpy as np
import pytest

import pattern_oracle as PO
import phrase_oracle as O
import postings_range as R
from phrase_fixtures import assert_same, index_to_csr, make_segment, native_batch, oracle_batch
from stract_b200.bm25 import (ABSENT_TERM, NO_TERM, PART_ANCHOR, PART_TERM, PART_WILDCARD, SegmentReader, TopDocs,
                              encode_postings, id_to_fieldnorm, pattern_docsets)

pytestmark = pytest.mark.gpu

MEDIUM = (1 << 22) + 12_345
KIND = {"T": PART_TERM, "*": PART_WILDCARD, "|": PART_ANCHOR}
# the offset each role takes in a phrase next to the anchor (its positions relative to the anchor's)
NATURAL = {"anchor": 0, "plus1": 1, "plus2": 2, "near1": 1, "near2": 1, "near3": 1, "df128": 1, "df129": 1, "df256": 1,
           "df257": 1, "vint": 1, "wrap_a": 0, "wrap_b": 1, "wrap_c": 2, "big_a": 0, "big_b": 1}
GROUPS = [("anchor", "plus1", "plus2"), ("anchor", "near1", "near2", "near3"),
          ("anchor", "plus1", "df128", "df129", "df256", "df257", "vint"), ("wrap_a", "wrap_b", "wrap_c"), ("big_a", "big_b")]


def make(seed, max_doc, counts=True):
    """the positional range index after its self-check, as a device segment with its token counts attached (`counts`:
    a u64 per document, 17 GB at max_doc 2^31 - 2, so the near-limit index goes without)"""
    fx = R.positional_range_index(seed, max_doc)
    fx["produced"] = R.positional_self_check(fx)
    fx["seg"] = make_segment(fx)
    if counts:
        fx["seg"].attach_token_counts(R.token_counts(fx))
    fx["csr"] = index_to_csr(fx)
    return fx


def phrase_groups(seg, rows, budget_mb):
    """how many candidate groups a phrase batch makes under a budget: rows packed in order while the rarest terms' doc
    freqs fit budget / (12 + 12 * width) entries (the candidate records of bm25.cu's run_phrase)"""
    cap = max((budget_mb << 20) // (12 + 12 * rows.shape[1]), 1)
    groups, used = 1, 0
    for r in rows:
        real = [int(t) for t in r if t != NO_TERM]
        df = 0 if ABSENT_TERM in real else min(int(seg.doc_freq[t]) for t in real)
        if used and used + df > cap:
            groups += 1; used = 0
        used += df
    return groups


def phrase_rows(fx, rng, nq, width=8):
    """phrases of 2..width terms drawn (with repeats: duplicate terms) from one group, in offset order, the offsets
    sometimes stretched; an ABSENT_TERM now and then; every fixed case of the fixture first"""
    ro = fx["roles"]
    fixed = [("anchor", "plus1"), ("anchor", "plus1", "plus2"), ("anchor", "near3"), ("wrap_a", "wrap_b", "wrap_c"),
             ("big_a", "big_b"), ("anchor", "df257", "plus2"), ("anchor", "vint")]
    rows = np.full((nq + len(fixed), width), NO_TERM, np.uint32); offs = np.zeros(rows.shape, np.uint32)
    for q in range(rows.shape[0]):
        if q < len(fixed):
            names = list(fixed[q])
        else:
            g = GROUPS[int(rng.integers(0, len(GROUPS)))]
            names = sorted(rng.choice(g, int(rng.integers(2, width + 1))).tolist(), key=lambda n: NATURAL[n])
        o = np.array([NATURAL[n] for n in names], np.int64)
        if q >= len(fixed) and rng.random() < 0.3:
            o = o + np.cumsum(rng.integers(0, 2, o.size))
        rows[q, :len(names)] = [ro[n] for n in names]
        offs[q, :len(names)] = o
        if q >= len(fixed) and rng.random() < 0.05:
            rows[q, len(names) - 1] = ABSENT_TERM
    return rows, offs


def native_expected(fx, rows, offs, slops, scoring, k):
    """the native oracle's answer, with the weights and tf cache the library derives from the segment"""
    seg = fx["seg"]
    n = seg.max_doc
    cache = O.tf_cache(seg.average_fieldnorm, [id_to_fieldnorm(i) for i in range(256)])
    ws = []
    for q in range(rows.shape[0]):
        real = [int(t) for t in rows[q] if t != NO_TERM]
        ws.append(O.bm25_weight_for_terms([0 if t == ABSENT_TERM else int(seg.doc_freq[t]) for t in real], n))
    return native_batch(fx["csr"], rows, offs, slops, ws, cache, scoring, k, threads=8)


def check_phrases(fx, rng, nq, slops=(0, 1, 3, 300), ks=(1, 10, 4096), python_rows=8, monkeypatch=None):
    """search_phrase_batch against the native oracle on every row, and against the Python oracle on the first rows; again
    with a 1 MB candidate budget when monkeypatch is given, on the rows repeated until they make at least six candidate
    groups.  Returns the matches seen."""
    seg = fx["seg"]
    rows0, offs0 = phrase_rows(fx, rng, nq)
    seen = 0
    for budget in ((None, "1") if monkeypatch is not None else (None,)):
        rows, offs = rows0, offs0
        if budget:
            monkeypatch.setenv("SB200_PHRASE_BUDGET_MB", budget)
            rep = 1
            while phrase_groups(seg, np.tile(rows0, (rep, 1)), 1) < 6:
                rep += 1
            rows, offs = np.tile(rows0, (rep, 1)), np.tile(offs0, (rep, 1))
        for slop in slops:
            sl = np.full(rows.shape[0], slop, np.uint32)
            for scoring in (True, False):
                for k in ks:
                    d, s, n = TopDocs.with_limit(k).search_phrase_batch(seg, rows, offs, sl, scoring)
                    ed, es, en = native_expected(fx, rows, offs, sl, scoring, k)
                    for q in range(rows.shape[0]):
                        m = int(n[q])
                        assert m == int(en[q]), (slop, scoring, k, q, rows[q], m, int(en[q]))
                        assert np.array_equal(d[q, :m], ed[q, :m]), (slop, scoring, k, q)
                        assert np.array_equal(s[q, :m].view(np.uint32), es[q, :m].view(np.uint32)), (slop, scoring, k, q)
                    seen += int(n.sum())
                    if budget is None and k == ks[-1]:
                        p = slice(0, python_rows)
                        assert_same((d[p], s[p], n[p]), oracle_batch(fx, rows[p], offs[p], sl[p], scoring, k))
    if monkeypatch is not None:
        monkeypatch.delenv("SB200_PHRASE_BUDGET_MB")
    # the fixed rows reach what they are there for: wide positions, the u32 wrap, the tf 2^16 + 1 posting
    d, _, n = TopDocs.with_limit(4096).search_phrase_batch(seg, rows0[:5], offs0[:5], np.full(5, 3, np.uint32))
    anchor = fx["terms"][fx["roles"]["anchor"]]
    last = {int(a): int(p[-1]) for a, p in zip(anchor["docs"], anchor["positions"])}
    assert max(last[int(x)] for x in d[0, :n[0]]) >= 1 << 31
    assert n[3] > 0 and n[4] == 10
    return seen


def pattern_expected(fx, parts, terms):
    """PatternWeight's docset from the input positions: the documents that hold every term and pass
    NormalPatternScorer::pattern_match (pattern_oracle.normal_pattern_match_pos) with their token count"""
    if any(t is None for t in terms):
        return np.zeros(0, np.uint32)
    tl = fx["terms"]
    common = tl[terms[0]]["docs"]
    for t in terms[1:]:
        common = np.intersect1d(common, tl[t]["docs"], assume_unique=True)
    out = []
    for doc in common:
        pos = [[int(x) for x in tl[t]["positions"][int(np.searchsorted(tl[t]["docs"], doc))]] for t in terms]
        if PO.normal_pattern_match_pos(pos, parts, R.token_count(fx, int(doc))):
            out.append(int(doc))
    return np.array(out, np.uint32)


def fixed_patterns(fx):
    ro = fx["roles"]
    a, p1, p2, n3 = ro["anchor"], ro["plus1"], ro["plus2"], ro["near3"]
    wa, wb, wc, ba, bb = ro["wrap_a"], ro["wrap_b"], ro["wrap_c"], ro["big_a"], ro["big_b"]
    pats = [(["T", "T"], [a, p1]), (["T", "T", "T"], [a, p1, p2]), (["T", "*", "T"], [a, n3]), (["T", "*", "T"], [a, p2]),
            (["|", "T", "T"], [a, p1]), (["|", "T"], [wa]), (["T", "|"], [wc]), (["|", "T", "*", "T", "|"], [wa, wc]),
            (["T"], [a]), (["T"], [ba]), (["T"], [None]), (["T", "T"], [a, None]), (["T", "T"], [ba, bb]),
            (["T", "T"], [a, a]), (["T", "*", "T", "T"], [a, p1, p2]), (["*", "T", "*"], [n3]),
            (["T", "T", "T", "T", "T", "T", "T", "T"], [a, p1, p2, p1, p2, a, p1, p2])]
    for name in ("anchor", "plus1", "plus2", "near1", "df256", "vint", "wrap_c", "big_a"):   # end anchors
        pats += [(["*", "T", "|"], [ro[name]]), (["T", "|"], [ro[name]])]
    pats += [(["T", "T", "|"], [a, p1]), (["T", "*", "T", "|"], [a, p2])]
    return pats


def check_patterns(fx, anchors=True):
    """pattern_docsets against the pattern oracle on the input positions: wildcards (u32::MAX slop), start and end
    anchors at wide positions, one-term patterns (every posting a candidate), absent and duplicate terms, the tf 2^16 + 1
    posting.  `anchors=False`: only the patterns that need no token counts."""
    seg = fx["seg"]
    pats = [p for p in fixed_patterns(fx) if anchors or "|" not in p[0]]
    rows = [([KIND[x] for x in parts], [ABSENT_TERM if t is None else t for t in terms]) for parts, terms in pats]
    wide_end = matched = 0
    got = pattern_docsets(seg, rows)
    for (parts, terms), ds in zip(pats, got):
        want = pattern_expected(fx, parts, terms)
        assert np.array_equal(ds.docs(), want), (parts, terms, ds.count(), want.size)
        assert ds.count() == want.size
        matched += want.size
        if parts[-1] == "|":
            wide_end += sum(R.token_count(fx, int(d)) > 1 << 30 for d in want)
        ds.close()
    assert matched > 0
    assert wide_end > 0 or not anchors, "an end anchor matched at a position above 2^30"


@pytest.fixture(scope="module")
def positional():
    fx = make(61, MEDIUM)
    yield fx
    fx["seg"].close()


def test_phrases_medium(positional, monkeypatch):
    assert check_phrases(positional, np.random.default_rng(1), 40, monkeypatch=monkeypatch) > 0


def test_patterns_medium(positional):
    check_patterns(positional)


def _free_device_bytes():
    import torch
    return torch.cuda.mem_get_info()[0]


def test_positions_beyond_4gib():
    """A term whose bit-packed positions pass 4 GiB: read_positions windows on both sides of the 4 GiB mark equal the
    delta array, and a phrase whose only candidates lie past it equals the oracle run on just those postings with the real
    doc_freqs.  Prints the time of each stage and the peak host memory."""
    need = 12 << 30
    if _free_device_bytes() < need:
        pytest.skip(f"needs {need >> 30} GiB of free device memory for a 5.4 GB positions file")
    t0 = time.time()
    h = R.huge_positions_term(71)
    stages = [("build", time.time() - t0)]
    t = time.time()
    ids = h["ids"]
    data, infos = encode_postings(h["docs"], h["tfs"], ids, 1.0, record_option=2)
    seg = SegmentReader(data, infos, ids, record_option=2, total_num_tokens=h["total"], positions=h["pos"],
                        positions_ranges=(h["po"], h["pl"]))
    stages.append(("attach", time.time() - t))
    t = time.time()
    deltas, late, lo = h["deltas"], h["late"], h["late_off"]

    def want(a, n):
        if a + n <= deltas.size:
            return deltas[a:a + n]
        return np.concatenate([deltas[a:], late[:a + n - deltas.size]]) if a < deltas.size else late[a - deltas.size:a - deltas.size + n]

    mark = 1 << 30   # value index of byte 4 GiB in the term's block data
    windows = [(0, 300), (mark - 1000, 999), (mark - 200, 700), (mark, 128), (mark + 77, 5000), (lo - 128 * 3 - 5, 500),
               (lo - 64, 64 + late.size), (lo, late.size), (lo + 100, 200), (lo + late.size - 70, 70), (deltas.size // 2 + 3, 4096)]
    for a, n in windows:
        assert np.array_equal(seg.read_positions(0, a, n), want(a, n)), (a, n)
    stages.append(("read", time.time() - t))
    t = time.time()
    rows = np.array([[0, 1]], np.uint32); offs = np.array([[0, 1]], np.uint32)
    dfs = [[int(seg.doc_freq[0]), int(seg.doc_freq[1])]]
    n_match = {}
    for slop in (0, 1, 3):
        sl = np.array([slop], np.uint32)
        for scoring in (True, False):
            got = TopDocs.with_limit(10).search_phrase_batch(seg, rows, offs, sl, scoring)
            exp = oracle_batch(h["index"], rows, offs, sl, scoring, 10, total_docs=seg.max_doc, avg=seg.average_fieldnorm, dfs=dfs)
            assert_same(got, exp)
            n_match[slop] = int(got[2][0])
    assert 0 < n_match[0] < n_match[3], n_match
    stages.append(("phrase", time.time() - t))
    t = time.time()
    # CleanBody min_slop (k_wp_slop) of the late documents, whose positions are read past the 4 GiB mark
    from stract_b200.bm25 import MultiFieldSignalComputer, SignalTable
    from stract_b200.ranking_pipeline import U32_MAX, min_slop
    comp = MultiFieldSignalComputer({"Title": seg, "CleanBody": seg}, {"Bm25Title", "Bm25CleanBody"},
                                    SignalTable([np.zeros(seg.max_doc)]), [("HostCentrality", 0, 1.0)])
    sf = np.array([[0, 0, 1, 1]], np.uint8); st = np.array([[0, 1, 0, 1]], np.uint32)
    late = h["index"]["terms"]
    docs = np.array([late[0]["docs"]], np.uint32)
    wp = comp.ranking_webpages(sf, st, docs, np.array([docs.shape[1]], np.uint32))
    for i, d in enumerate(docs[0]):
        lists = [[int(x) for x in t["positions"][int(np.searchsorted(t["docs"], d))]] if d in t["docs"] else [] for t in late]
        want = min_slop(lists)
        assert tuple(int(x) for x in wp.min_slop[0, i]) == (want, want), (int(d), wp.min_slop[0, i], want)
    assert any(int(x) < U32_MAX for x in wp.min_slop[0, :, 1])
    stages.append(("min_slop", time.time() - t))
    seg.close()
    print("beyond 4 GiB:", ", ".join(f"{n} {s:.1f} s" for n, s in stages),
          f"; peak host RSS {resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20:.2f} GB")


# ---- multi-field signals, optic rules, query plans and recall webpages over range and positional fields -------------------
MF = ["Title", "CleanBody", "Url", "TitleBigrams"]     # Title / CleanBody: positional fixtures; Url / TitleBigrams: range_index
MF_ENABLED = {"Bm25F", "Bm25Title", "TitleCoverage", "Bm25TitleBigrams", "Bm25CleanBody", "CleanBodyCoverage", "IdfSumUrl"}


def _positional_pair(fx):
    """(oracle Segment, device segment with positions and token counts) of a positional fixture"""
    import test_bm25_gpu as T
    from stract_b200.bm25 import encode_positions
    terms = fx["terms"]
    tfs = [np.array([p.size for p in t["positions"]], np.uint32) for t in terms]
    oseg, seg = T.build([t["docs"] for t in terms], tfs, None, 2, fieldnorm_ids=fx["fieldnorm_ids"])
    off = np.concatenate([[0], np.cumsum([t["docs"].size for t in terms])])
    pos, po, pl = encode_positions(np.concatenate([p for t in terms for p in t["positions"]]), np.concatenate(tfs), off)
    seg.attach_positions(pos, (po, pl))
    seg.attach_token_counts(R.token_counts(fx))
    return oseg, seg


def make_fields(seed, max_doc, big=True):
    """Title / CleanBody: positional_range_index (record option 2, positions attached); Url: range_index with record
    option 1 (tfs up to 2^32 - 1, every fieldnorm code, the 70 000-posting term when `big`); TitleBigrams: range_index with
    record option 2.  Each after its self-check.  Returns (pairs {name: (oracle Segment, segment)}, fixtures, computer,
    numeric columns)."""
    import test_bm25_gpu as T
    fxs, pairs = {}, {}
    for i, name in enumerate(("Title", "CleanBody")):
        fx = R.positional_range_index(seed + i, max_doc)
        fx["produced"] = R.positional_self_check(fx)
        fxs[name], pairs[name] = fx, _positional_pair(fx)
    for i, (name, ro, b) in enumerate((("Url", 1, big), ("TitleBigrams", 2, False))):
        fx = R.range_index(seed + 2 + i, max_doc, ro, b)
        oseg, seg = T.build(fx["docs"], fx["tfs"], None, ro, fieldnorm_ids=fx["ids"])
        fx["produced"] = R.self_check(fx, oseg.postings_bytes(), oseg.term_infos())
        fxs[name], pairs[name] = fx, (oseg, seg)
    cols = [np.random.default_rng(seed).random(max_doc)]
    from stract_b200.bm25 import MultiFieldSignalComputer, SignalTable
    comp = MultiFieldSignalComputer({n: pairs[n][1] for n in MF}, MF_ENABLED, SignalTable(cols), [("HostCentrality", 0, 1.0)])
    assert comp.names == MF
    return pairs, fxs, comp, cols


def mf_slots(fxs, rng, nq, ns):
    """queries of up to ns slots in field order: Title / CleanBody terms from one positional group (the same roles in
    both fields), Url / TitleBigrams terms from one range group; unknown terms (NO_TERM) now and then.  The last query is
    the 70 000-posting Url term with one Title term (a query that term dominates) when Url has it."""
    sf = np.full((nq, ns), 0xFF, np.uint8); st = np.full((nq, ns), NO_TERM, np.uint32)
    ro = fxs["Title"]["roles"]
    for q in range(nq):
        g = GROUPS[int(rng.integers(0, len(GROUPS)))]
        names = rng.choice(g, int(rng.integers(1, 4))).tolist()
        x = 0
        for f, fname in enumerate(MF):
            if f < 2:
                ts = [ro[n] for n in names]
            else:
                grp = fxs[fname]["groups"][int(rng.integers(0, len(fxs[fname]["groups"])))]
                ts = [int(t) for t in rng.choice(grp, int(rng.integers(1, 3)))]
            for t in ts:
                if x < ns - (len(MF) - 1 - f):
                    sf[q, x] = f; st[q, x] = NO_TERM if rng.random() < 0.08 else t; x += 1
        while x < ns and ns > 8:                             # fill up to the 9..16-slot kernel
            f = int(rng.integers(0, 2)); sf[q, x] = f; st[q, x] = ro[rng.choice(g)]; x += 1
    big = [t for t in range(len(fxs["Url"]["docs"])) if fxs["Url"]["docs"][t].size > 65_536]
    if big:
        sf[-1] = 0xFF; st[-1] = NO_TERM
        sf[-1, :2] = (0, 2); st[-1, :2] = (ro["anchor"], big[0])
    return sf, st


def check_multi_field(mf, rng, nq, ks=(10, 1000), widths=(8, 16)):
    """top_docs_batch (k_sig_multi: Bm25 per field, Bm25F, coverage, idf_sum) against oracle.multi_signal_topk, at 8 and
    16 slots per query (both TMAX kernels); f64 totals and doc order bit for bit"""
    import test_multi_signal_gpu as MS
    pairs, fxs, comp, cols = mf
    for ns in widths:
        sf, st = mf_slots(fxs, rng, nq, ns)
        for k in ks:
            MS.check_against_oracle(comp, pairs, cols, sf, st, k, None)


def _rule_docsets(mf, rng):
    """docsets from postings of every field, an AND / OR of them and pattern docsets of the positional Title, with their sets"""
    from stract_b200.bm25 import Docset
    pairs, fxs, comp, cols = mf
    ro = fxs["Title"]["roles"]
    docsets, sets = [], []
    for f in MF:
        terms = fxs[f]["terms"] if f in ("Title", "CleanBody") else [{"docs": d} for d in fxs[f]["docs"]]
        for t in rng.choice(len(terms), 4, replace=False):
            docsets.append(Docset.from_postings(pairs[f][1], int(t))); sets.append(set(terms[int(t)]["docs"].tolist()))
    for op, fn in (("and", set.intersection), ("or", set.union)):
        idx = [int(x) for x in rng.choice(len(docsets), 3, replace=False)]
        docsets.append(Docset.combine(op, [docsets[i] for i in idx])); sets.append(fn(*[sets[i] for i in idx]))
    pats = [(["T", "T"], [ro["anchor"], ro["plus1"]]), (["T", "*", "T", "|"], [ro["anchor"], ro["plus2"]]), (["T"], [ro["big_a"]])]
    for (parts, terms), ds in zip(pats, pattern_docsets(pairs["Title"][1], [([KIND[x] for x in p], t) for p, t in pats])):
        docsets.append(ds); sets.append(set(pattern_expected(fxs["Title"], parts, terms).tolist()))
    for d, s in zip(docsets, sets):
        assert np.array_equal(d.docs(), np.array(sorted(s), np.uint32))
    return docsets, sets


def check_optic(mf, rng, nq, k=100):
    """top_docs_batch(optic=) against the multi-field oracle's every-candidate totals filtered and boosted by
    pattern_oracle.optic_topk: rules, exclude and require over posting, combined and pattern docsets"""
    import test_optic_gpu as TO
    from stract_b200.bm25 import OpticTables
    pairs, fxs, comp, cols = mf
    docsets, sets = _rule_docsets(mf, rng)
    nd = len(docsets)
    sf, st = mf_slots(fxs, rng, nq, 8)
    rules = [[(int(rng.integers(0, nd)), float(rng.choice([-4.0, -1.0, 0.5, 2.0, 3.0]))) for _ in range(q % 4)] for q in range(nq)]
    exclude = [None if q % 3 == 0 else int(rng.integers(0, nd)) for q in range(nq)]
    require = [None if q % 5 < 2 else int(rng.integers(0, nd)) for q in range(nq)]
    tables = OpticTables(docsets, rules, exclude, require)
    docs, totals, n_out = comp.top_docs_batch(sf, st, k, optic=tables)
    want = TO.oracle_recall(comp, pairs, cols, sf, st, k, tables, sets)
    for q in range(nq):
        n = int(n_out[q])
        assert n == len(want[q]), (q, n, len(want[q]))
        assert np.array_equal(docs[q, :n], np.array([d for _, d in want[q]], np.uint32)), q
        assert np.array_equal(totals[q, :n].view(np.uint64), np.array([t for t, _ in want[q]], np.float64).view(np.uint64)), q


def plan_programs(fxs, rng, nq, n_range_terms):
    """programs of 1..4 TERM / PHRASE leaves under Must / Should / MustNot over the four fields; phrase rows on Title"""
    import test_recall_plan_gpu as TP
    from stract_b200.bm25 import PLAN_BOOL, PLAN_PHRASE, PLAN_TERM
    M, S, N = TP.M, TP.S, TP.N
    ro = fxs["Title"]["roles"]
    phrases = [([ro["anchor"], ro["plus1"]], [0, 1], 0), ([ro["anchor"], ro["near3"]], [0, 1], 3),
               ([ro["wrap_a"], ro["wrap_b"], ro["wrap_c"]], [0, 1, 2], 3), ([ro["big_a"], ro["big_b"]], [0, 1], 0),
               ([ro["anchor"], ro["plus1"], ro["plus2"]], None, 0), ([ro["anchor"], ABSENT_TERM], [0, 1], 0)]
    progs = []
    for q in range(nq):
        prog, n = [], int(rng.integers(1, 5))
        for _ in range(n):
            occ = int(rng.choice([M, M, S, S, N]))
            x = rng.random()
            if x < 0.35:
                prog.append((PLAN_PHRASE, occ, 0, 0, int(rng.integers(0, len(phrases)))))
            elif x < 0.7:
                f = int(rng.integers(0, 2))
                prog.append((PLAN_TERM, occ, 0, f, int(ro[rng.choice(list(ro))])))
            else:
                f = int(rng.integers(2, 4))
                prog.append((PLAN_TERM, occ, 0, f, int(rng.integers(0, n_range_terms[f - 2]))))
        prog.append((PLAN_BOOL, M, n, 0, 0))
        progs.append(prog)
    progs.append([(PLAN_PHRASE, M, 0, 0, 2)])                 # the wrap phrase alone (phrase_exists: no carrying slop)
    progs.append([(PLAN_TERM, M, 0, 0, ro["anchor"]), (PLAN_PHRASE, S, 0, 0, 0), (PLAN_BOOL, M, 2, 0, 0)])
    return progs, phrases


def check_plans(mf, rng, nq, k=200, monkeypatch=None):
    """recall_plan_docs (k_plan_recall, pl_seek_at) with TERM and PHRASE leaves against plan_oracle.program_docs fed with
    the input docs and the phrase oracle; top_docs_batch(plan=) against the multi-field oracle's totals over the plan's
    docs; again with 1 MB AND3 / plan budgets (several groups) when monkeypatch is given"""
    import plan_oracle as PLO
    import test_optic_gpu as TO
    import test_recall_plan_gpu as TP
    from stract_b200.bm25 import OpticTables, RecallPlan, recall_plan_docs
    pairs, fxs, comp, cols = mf
    progs, phrases = plan_programs(fxs, rng, nq, [len(fxs["Url"]["docs"]), len(fxs["TitleBigrams"]["docs"])])
    plan = RecallPlan([pairs[n][1] for n in MF], progs, phrases)
    title = fxs["Title"]
    ps = [PLO.phrase_exists_docs(title, [None if t == ABSENT_TERM else t for t in terms],
                                 list(range(len(terms))) if offs is None else offs, sl) for terms, offs, sl in phrases]
    assert ps[0] and ps[3], "phrase leaves at wide positions and on the tf 2^16 + 1 posting match"
    post = [[t["docs"] for t in fxs["Title"]["terms"]], [t["docs"] for t in fxs["CleanBody"]["terms"]],
            fxs["Url"]["docs"], fxs["TitleBigrams"]["docs"]]
    want_sets = [PLO.program_docs(p, post, ps) for p in progs]
    nqq = len(progs)
    sf, st = mf_slots(fxs, rng, nqq, 8)
    for budget in ((None, "1") if monkeypatch is not None else (None,)):
        if budget:
            monkeypatch.setenv("SB200_AND3_BUDGET_MB", budget); monkeypatch.setenv("SB200_PLAN_BUDGET_MB", budget)
        got = recall_plan_docs(plan)
        for q, prog in enumerate(progs):
            assert np.array_equal(got[q], np.array(want_sets[q], np.uint32)), (q, prog, got[q].size, len(want_sets[q]))
        docs, totals, n_out = comp.top_docs_batch(sf, st, k, plan=plan)
        union = TO.oracle_recall(comp, pairs, cols, sf, st, comp.readers[0].max_doc, OpticTables([], [[] for _ in range(nqq)]), [])
        for q in range(nqq):
            tot = {d: t for t, d in union[q]}
            cand = [(d, tot[d] if d in tot else TP.zero_text_total(comp, cols, d)) for d in want_sets[q]]
            want = PO.optic_topk(cand, k)
            n = int(n_out[q])
            assert n == len(want), (q, n, len(want))
            assert np.array_equal(docs[q, :n], np.array([d for _, d in want], np.uint32)), q
            assert np.array_equal(totals[q, :n].view(np.uint64), np.array([t for t, _ in want], np.float64).view(np.uint64)), q
    if monkeypatch is not None:
        monkeypatch.delenv("SB200_AND3_BUDGET_MB"); monkeypatch.delenv("SB200_PLAN_BUDGET_MB")


def _webpage_oracle(mf):
    import webpage_oracle as WO
    pairs, fxs, comp, cols = mf
    fields = []
    for n in MF:
        fx = fxs[n]
        if n in ("Title", "CleanBody"):
            fields.append({"terms": fx["terms"], "ids": fx["fieldnorm_ids"]})
        else:
            fields.append({"terms": [{"docs": d, "tfs": t} for d, t in zip(fx["docs"], fx["tfs"])], "ids": fx["ids"]})
    ops = [(kind, comp.names.index(field) if field is not None else 0, chain, col, comp.coefficient(name, coef))
           for name, kind, field, chain, col, coef in comp.order.entries]
    return WO.Oracle(fields, comp.last_inputs["caches"], comp.k1, [np.float32(comp.field_coefficient(n)) for n in comp.names], ops, cols)


def check_webpages(mf, rng, nq, k=50):
    """ranking_webpages (k_wp_signals with WpPos, k_wp_slop) against webpage_oracle.Oracle: values, scores, boost and both
    min_slops bit for bit for each query's top-k plus documents near max_doc - 1, the tf 2^16 + 1 document, the wrap
    documents and documents no slot holds; the top-k totals rebuilt from the scores; recall_stage over the device pages
    equals recall_stage over the oracle's"""
    import webpage_oracle as WO
    from stract_b200 import ranking_pipeline as RP
    pairs, fxs, comp, cols = mf
    max_doc = comp.readers[0].max_doc
    sf, st = mf_slots(fxs, rng, nq, 16)
    td, tt, tn = comp.top_docs_batch(sf, st, k)
    title = fxs["Title"]
    ro = title["roles"]
    special = [int(title["terms"][ro["big_a"]]["docs"][200]), max_doc - 1, max_doc - 2, max_doc - 3] + \
        [int(d) for d in title["terms"][ro["wrap_c"]]["docs"][:3]] + [int(d) for d in title["end_anchored"][:3]]
    lists = []
    for q in range(nq):
        d = td[q, :tn[q]].tolist() + special + rng.integers(0, max_doc, 6).tolist()
        rng.shuffle(d)
        lists.append(d)
    n = np.array([len(x) for x in lists], np.uint32)
    docs = np.zeros((nq, int(n.max())), np.uint32)
    for q, x in enumerate(lists):
        docs[q, :len(x)] = x
    wp = comp.ranking_webpages(sf, st, docs, n)
    O = _webpage_oracle(mf)
    numeric = [o for o, e in enumerate(comp.order.entries) if e[1] == WO.OP_NUMERIC]
    bits = lambda x: np.asarray(x, np.float64).view(np.uint64)
    for q in range(nq):
        text = [(x, int(sf[q, x]), int(st[q, x])) for x in range(sf.shape[1]) if sf[q, x] != 0xFF]
        slots = [(f, o) for _, f, o in text]
        idf = [comp.last_inputs["idf"][q][x] for x, _, _ in text]
        idf_f = [comp.last_inputs["idf_f"][q][x] for x, _, _ in text]
        known = {int(a): t for a, t in zip(td[q, :tn[q]], tt[q, :tn[q]])}
        for i, d in enumerate(lists[q]):
            v, s, b, sl = O.page(d, slots, idf, idf_f, dist=(0, 1))
            for o in numeric:
                v[o] = np.nan
            assert np.array_equal(bits(wp.values[q, i]), bits(v)), (q, i, d)
            assert np.array_equal(bits(wp.scores[q, i]), bits(s)), (q, i, d)
            assert bits(wp.boosts[q, i]) == bits(b), (q, i, d)
            assert tuple(int(x) for x in wp.min_slop[q, i]) == sl, (q, i, d, wp.min_slop[q, i], sl)
            if d in known:
                assert bits(O.total(wp.scores[q, i], wp.boosts[q, i])) == bits(known[d]), (q, i, d)
        m = int(tn[q])
        inbound = {d: float(np.float64(d % 1009) / 1009.0) for d in lists[q]}
        got = RP.recall_stage(RP.pages_from_webpages(wp, q, np.array(lists[q], np.uint32), len(lists[q]),
                                                     np.zeros(len(lists[q]))), RP.default_coefficients(), inbound)
        want_pages = []
        for d in lists[q]:
            v, s, b, sl = O.page(d, slots, idf, idf_f, dist=(0, 1))
            for o in numeric:
                v[o] = np.nan
            p = RP.Page(int(d), {name: (v[o], s[o]) for o, name in enumerate(wp.names)}, 0.0, b)
            p.min_slop = sl
            want_pages.append(p)
        want = RP.recall_stage(want_pages, RP.default_coefficients(), inbound)
        assert [p.key for p in got] == [p.key for p in want], q
        assert all(bits(a.score) == bits(b.score) and bits(a.boost) == bits(b.boost) for a, b in zip(got, want)), q
        assert m > 0 or not any(x != NO_TERM for x in st[q])


@pytest.fixture(scope="module")
def fields():
    return make_fields(81, MEDIUM)


def test_multi_field_signals(fields):
    check_multi_field(fields, np.random.default_rng(11), 24)


def test_multi_field_optic(fields):
    check_optic(fields, np.random.default_rng(12), 16)


def test_plan_docsets_and_recall(fields, monkeypatch):
    check_plans(fields, np.random.default_rng(13), 40, monkeypatch=monkeypatch)


def test_recall_webpages(fields):
    check_webpages(fields, np.random.default_rng(14), 16)


NEAR_LIMIT = (1 << 31) - 2


def test_near_limit_positional_index():
    """max_doc = 2^31 - 2: phrases, unanchored pattern docsets and plan docsets with TERM and PHRASE leaves on the
    positional index, doc ids up to 2^31 - 3.  No token counts (17 GB of u64) and so no anchored patterns; no
    multi-field top-k, whose SignalTable would need f64 columns of 17 GB.  Prints the time of each stage and the peak host
    memory."""
    import plan_oracle as PLO
    from stract_b200.bm25 import RecallPlan, recall_plan_docs
    t0 = time.time()
    fx = make(91, NEAR_LIMIT, counts=False)
    assert fx["produced"][2] >= 29
    stages = [("build", time.time() - t0)]
    rng = np.random.default_rng(15)
    t = time.time()
    check_phrases(fx, rng, 12, slops=(0, 3), ks=(10, 4096), python_rows=7)
    stages.append(("phrases", time.time() - t)); t = time.time()
    check_patterns(fx, anchors=False)
    stages.append(("patterns", time.time() - t)); t = time.time()
    progs, phrases = plan_programs({"Title": fx}, rng, 30, [1, 1])
    progs = [[n[:3] + (0,) + n[4:] for n in p] for p in progs]          # every leaf on the one segment
    plan = RecallPlan([fx["seg"]], progs, phrases)
    ps = [PLO.phrase_exists_docs(fx, [None if x == ABSENT_TERM else x for x in terms],
                                 list(range(len(terms))) if offs is None else offs, sl) for terms, offs, sl in phrases]
    post = [[x["docs"] for x in fx["terms"]]]
    got = recall_plan_docs(plan)
    for q, prog in enumerate(progs):
        assert np.array_equal(got[q], np.array(PLO.program_docs(prog, post, ps), np.uint32)), (q, prog)
    stages.append(("plans", time.time() - t))
    fx["seg"].close()
    print("near-limit positional index:", ", ".join(f"{n} {s:.1f} s" for n, s in stages),
          f"; peak host RSS {resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20:.2f} GB")
