"""Optic rule benchmark: docset builds (sb200_pattern_docsets) and the multi-field recall stage with optic docsets
(sb200_multi_signal_topk_batch_optic), with parity against the plain oracle (tests/pattern_oracle.py, oracle/).

Index (seeded):
  body   the C4-shaped positions index of tools/phrase_bench.py (10 M docs, Zipf ranks <= 10 000, tf distinct positions per
         posting); its doc lengths are the token-count column.
  site   a no-tokenizer site field over the same docs: every doc gets one of 100 k sites, Zipf(1.1) distributed (one posting).
  recall the three-field index and 10 k-query batch of bench_bm25.run_multi (same seeds), opened over the same 10 M docs.
Timed (kernel ms = the library's CUDA-event time of the launches, median of --steps after --warmup):
  site_rules     1 000 Site("|site|") docsets (the FastSiteDomain posting-list path), one call
  body_patterns  50 body patterns of 2-4 terms with wildcards and start / end anchors, one call: candidates / s, positions / s;
                 roofline = (posting bytes of the terms + position bytes decoded + bitmap words written) / kernel time
  recall_*       the recall batch with 0 / 8 / 64 boost rules per query (site and body docsets, mixed boost / downrank), an exclude
                 of 100 blocked sites and a require (the OR of the 1 000 site rules), against the same batch through
                 sb200_multi_signal_topk_batch
Parity: the first body patterns and site rules against the oracle restatement, and the first recall queries (docs and f64
total bits) against the multi-field oracle with the optic filters and boosts applied on the host.  The card's name and power
limit are read in the same run.  One JSON line on stdout; exit status 1 on any mismatch."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from stract_b200 import bm25  # noqa: E402
from stract_b200.bm25 import PART_ANCHOR, PART_TERM, PART_WILDCARD, Docset, OpticTables, pattern_docsets  # noqa: E402

HBM_GBS = 3350.0


def med_kernel(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    kms, out = [], None
    for _ in range(steps):
        out = fn()
        kms.append(out[1]["kernel_ms"])
    return out, float(np.median(kms))


def body_patterns(rng, n):
    """2-4 terms of ranks log-uniform in [10, 2 000], wildcards between terms, start / end anchors."""
    out = []
    for _ in range(n):
        nt = int(rng.integers(2, 5))
        terms = [int(np.exp(rng.uniform(np.log(10), np.log(2000)))) - 1 for _ in range(nt)]
        parts = []
        for i in range(nt):
            if i and rng.random() < 0.4:
                parts.append(PART_WILDCARD)
            parts.append(PART_TERM)
        if rng.random() < 0.3:
            parts.insert(0, PART_ANCHOR)
        if rng.random() < 0.3:
            parts.append(PART_ANCHOR)
        out.append((parts, terms))
    return out


def oracle_pattern(ix, parts, terms):
    import pattern_oracle as PO
    to = ix["term_off"]; po = ix["pos_off"]
    lists = [ix["docs"][int(to[t]):int(to[t + 1])] for t in terms]
    cand = lists[0]
    for l in lists[1:]:
        cand = np.intersect1d(cand, l, assume_unique=True)
    sym = ["T" if p == PART_TERM else ("*" if p == PART_WILDCARD else "|") for p in parts]
    out = []
    for d in cand:
        pos = []
        for t, l in zip(terms, lists):
            i = int(to[t]) + int(np.searchsorted(l, d))
            pos.append(ix["positions"][int(po[i]):int(po[i + 1])].tolist())
        if PO.normal_pattern_match_pos(pos, sym, int(ix["lens"][d])):
            out.append(int(d))
    return np.array(out, np.uint32)


def oracle_recall(comp, osegs, cols, sf, st, k, rules, ex, rq, max_doc):
    """Every candidate's total from the multi-field oracle, then the optic filters and boosts (vectorised, rule order)."""
    import oracle
    coefs = [np.float32(comp.field_coefficient(n)) for n in comp.names]
    ops = [(kind, comp.names.index(field) if field is not None else 0, chain, col, comp.coefficient(name, coef))
           for name, kind, field, chain, col, coef in comp.order.entries]
    od, ot = oracle.multi_signal_topk(osegs, comp.last_inputs["caches"], [1.2] * 3, coefs, sf, st, comp.last_inputs["idf"][0],
                                      comp.last_inputs["idf_f"][0], ops, cols, max_doc)
    keep = np.ones(od.size, bool)
    if ex is not None:
        keep &= ~ex(od)
    if rq is not None:
        keep &= rq(od)
    od, ot = od[keep], ot[keep]
    if rules:
        down = np.zeros(od.size); up = np.zeros(od.size)
        for member, b in rules:
            hit = member(od)
            if b < 0.0:
                down[hit] += abs(b)
            else:
                up[hit] += b
        with np.errstate(divide="ignore"):   # np.where evaluates both branches; the division is used only where down > up
            ot = ot * np.where(down > up, 1.0 / (1.0 + (down - up)), (up - down) + 1.0)
    o = np.lexsort((od, -ot))[:k]
    return od[o], ot[o]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=10_000)
    ap.add_argument("--k", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=4, help="recall queries checked against the oracle")
    a = ap.parse_args()
    import bench_bm25 as BB
    import phrase_bench as PB
    t0 = time.perf_counter()
    N = a.docs
    ix = PB.synth_index(N, 2.0e6 * N / 10_000_000)
    ids = bm25.fieldnorms_to_ids(ix["lens"])
    total_tokens = int(bm25.fieldnorm_table()[ids].astype(np.uint64).sum())
    avg = np.float32(np.float32(total_tokens) / np.float32(N))
    data, infos = bm25.encode_postings_csr(ix["docs"], ix["tfs"], ix["term_off"], ids, avg, threads=PB.host_threads(), record_option=2)
    pbytes, po, pl = bm25.encode_positions(ix["positions"], ix["tfs"], ix["term_off"])
    body = bm25.SegmentReader(data, infos, ids, record_option=2, total_num_tokens=total_tokens, positions=pbytes, positions_ranges=(po, pl))
    body.attach_token_counts(ix["lens"].astype(np.uint64))
    plen = np.array([infos[i].postings_len for i in range(len(infos))], np.float64)
    rng = np.random.default_rng(11)
    n_sites = 100_000
    site_of = np.minimum(rng.zipf(1.1, N), n_sites) - 1
    site_of = np.unique(site_of, return_inverse=True)[1]   # sites without a document get no term
    n_sites = int(site_of.max()) + 1
    order = np.argsort(site_of, kind="stable").astype(np.uint32)
    s_off = np.zeros(n_sites + 1, np.uint64)
    np.cumsum(np.bincount(site_of, minlength=n_sites), out=s_off[1:])
    s_ids = bm25.fieldnorms_to_ids(np.ones(N, np.uint32))
    sdata, sinfos = bm25.encode_postings_csr(order, np.ones(N, np.uint32), s_off, s_ids, np.float32(1.0), threads=PB.host_threads())
    site = bm25.SegmentReader(sdata, sinfos, s_ids, total_num_tokens=N)
    gen_s = time.perf_counter() - t0
    result = {"workload": f"{N} docs: body positions index ({ix['docs'].size} postings, {ix['positions'].size} positions), "
                          f"site field of {n_sites} Zipf sites, recall batch of {a.queries} queries top-{a.k}",
              "card": PB.card(), "gen_s": round(gen_s, 1), "batches": {}}
    green = True
    # ---- site rules: 1 000 posting-list docsets
    site_ids = np.unique(np.minimum(rng.zipf(1.3, 4000), n_sites) - 1)[:1000]
    site_ids = np.concatenate([site_ids, np.setdiff1d(np.arange(n_sites), site_ids)[:1000 - site_ids.size]])
    site_rows = [([PART_TERM], [int(s)]) for s in site_ids]
    (sd, st), kern = med_kernel(lambda: pattern_docsets(site, site_rows, return_stats=True), a.steps, a.warmup)
    nw = (N + 31) // 32
    post = int(sum(int(site.doc_freq[s]) for s in site_ids))
    alg = float(sum(sinfos[int(s)].postings_len for s in site_ids)) + 4.0 * nw * len(site_ids)
    bad = sum(int(not np.array_equal(sd[i].docs(), np.sort(order[int(s_off[s]):int(s_off[s + 1])]))) for i, s in enumerate(site_ids[:20]))
    result["batches"]["site_rules"] = {"rules": len(site_ids), "kernel_ms": kern, "postings": post, "postings_per_s": post / (kern * 1e-3),
                                       "roofline": {"alg_bytes": alg, "achieved_gbs": alg / (kern * 1e-3) / 1e9, "peak_gbs": HBM_GBS},
                                       "parity": {"rules": 20, "n_mismatch": bad, "green": bad == 0}}
    green &= bad == 0
    # ---- body patterns
    pats = body_patterns(rng, 50)
    (bd, st), kern = med_kernel(lambda: pattern_docsets(body, pats, return_stats=True), a.steps, a.warmup)
    alg = float(sum(plen[t].sum() for _, t in pats)) + st["position_bytes"] + 4.0 * nw * len(pats)
    bad = sum(int(not np.array_equal(bd[i].docs(), oracle_pattern(ix, *pats[i]))) for i in range(5))
    result["batches"]["body_patterns"] = {"patterns": len(pats), "kernel_ms": kern, "candidates": st["candidates"], "matches": st["matches"],
                                          "candidates_per_s": st["candidates"] / (kern * 1e-3), "positions_decoded": st["positions_decoded"],
                                          "positions_per_s": st["positions_decoded"] / (kern * 1e-3),
                                          "roofline": {"alg_bytes": alg, "achieved_gbs": alg / (kern * 1e-3) / 1e9, "peak_gbs": HBM_GBS,
                                                       "frac": alg / (kern * 1e-3) / 1e9 / HBM_GBS},
                                          "parity": {"patterns": 5, "n_mismatch": bad, "green": bad == 0}}
    green &= bad == 0
    # ---- recall stage
    names = ["Title", "CleanBody", "Url"]
    rixs = [BB.synth_index(N, 2.0e6 * N / 10_000_000 * f, seed=1234 + 17 * i) for i, f in enumerate((0.25, 1.0, 0.1))]
    r2 = np.random.default_rng(7)
    cols = [r2.random(N) ** 8, 1.0 / (1.0 + r2.integers(0, 1000, N).astype(np.float64))]
    segs = [bm25.SegmentReader(x["postings"], x["infos"], x["fieldnorm_ids"], total_num_tokens=x["total_num_tokens"]) for x in rixs]
    table = bm25.SignalTable(cols)
    enabled = {"Bm25F", "Bm25Title", "TitleCoverage", "Bm25CleanBody", "CleanBodyCoverage", "IdfSumUrl"}
    comp = bm25.MultiFieldSignalComputer(dict(zip(names, segs)), enabled, table, [("HostCentrality", 0, 2.5), ("FetchTimeMs", 1, 0.001)])
    q3 = BB.log_uniform_queries(a.queries, 3, seed=5)
    sf = np.tile(np.repeat(np.arange(3, dtype=np.uint8), 3), (a.queries, 1))
    stt = np.tile(q3, (1, 3)).astype(np.uint32)
    blocked = Docset.combine("or", sd[-100:])
    require = Docset.combine("or", sd)
    docsets = list(sd) + list(bd) + [blocked, require]
    ib, ir = len(docsets) - 2, len(docsets) - 1
    cand_rules = list(range(len(sd))) + list(range(len(sd), len(sd) + len(bd)))
    runs = {}

    def timed_batch(optic):
        def f():
            d, t, n, s = comp.top_docs_batch(sf, stt, a.k, return_stats=True, optic=optic)
            return (d, t, n), s
        return med_kernel(f, a.steps, a.warmup)

    _, kb = timed_batch(None)
    runs["recall_existing_entry"] = {"kernel_ms": kb}
    lists = {}

    def mask(i):
        """membership in docset i: a binary search in its document list"""
        if i not in lists:
            lists[i] = docsets[i].docs()
        docs = lists[i]

        def member(x):
            j = np.minimum(np.searchsorted(docs, x), max(docs.size - 1, 0))
            return (docs.size > 0) & (docs[j] == x) if docs.size else np.zeros(x.size, bool)
        return member

    osegs = []
    if a.sample:
        import oracle
        for x in rixs:
            o = oracle.Segment(x["fieldnorm_ids"], avg_fieldnorm=x["avg"])
            inf = x["infos"]; nt = len(inf)
            o.set_postings(x["postings"], [inf[i].postings_off for i in range(nt)], [inf[i].postings_len for i in range(nt)],
                           [inf[i].doc_freq for i in range(nt)])
            osegs.append(o)
    for nr in (0, 8, 64):
        rr = np.random.default_rng(100 + nr)
        rules = [[(int(rr.choice(cand_rules)), float(rr.choice([-3.0, -1.0, 1.0, 2.0, 5.0]))) for _ in range(nr)] for _ in range(a.queries)]
        tables = OpticTables(docsets, rules, [ib] * a.queries, [ir] * a.queries)
        ((d, t, n), _), kern = timed_batch(tables)
        entry = {"kernel_ms": kern, "kernel_ms_over_existing": kern / kb, "results": int(n.sum())}
        bad = 0
        if a.sample:
            for q in range(a.sample):
                comp.top_docs_batch(sf[q:q + 1], stt[q:q + 1], a.k)   # last_inputs of this query
                od, ot = oracle_recall(comp, osegs, cols, sf[q], stt[q], a.k, [(mask(i), b) for i, b in rules[q]], mask(ib), mask(ir), N)
                m = int(n[q])
                bad += int(m != od.size or not np.array_equal(d[q, :m], od) or not np.array_equal(t[q, :m].view(np.uint64), ot.view(np.uint64)))
            entry["parity"] = {"queries": a.sample, "n_mismatch": bad, "green": bad == 0}
            green &= bad == 0
        runs[f"recall_{nr}_rules"] = entry
    result["batches"].update(runs)
    result["parity_green"] = bool(green)
    print(json.dumps(result))
    return 0 if green else 1


if __name__ == "__main__":
    sys.exit(main())
