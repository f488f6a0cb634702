"""BM25 legs of bench.py: configs[3] (10M docs, 2-term AND, top-1000, 10k-query batch) and configs[4]
(100M docs, 5-term OR, Stract BM25 + linear signal combine, 10k-query batch) on one GPU.

Synthetic index (SURVEY.md 8d, seeded): vocabulary Zipf(1.0), df_r = round(2e6 / r) at 10M docs (x10 at 100M);
only ranks <= 10 000 are materialised because queries draw ranks from [10, 10 000]; a term's docs are a
uniform sorted subset drawn through geometric gaps (p = df/max_doc), tf ~ 1 + Geometric(0.6) capped at 255,
doc length ~ LogNormal(5.5, 0.8) -> fieldnorm id.  Posting lists are written in tantivy's byte format by the
library's host writer (sb200_postings_encode)."""
import time

import numpy as np

from stract_b200 import bm25


def synth_index(max_doc, df_scale, n_ranks=10_000, seed=1234, threads=16):
    rng = np.random.default_rng(seed)
    lens = np.minimum(np.maximum(1, rng.lognormal(5.5, 0.8, max_doc)), 2e9).astype(np.uint32)
    ids = bm25.fieldnorms_to_ids(lens)
    del lens
    total_tokens = int(bm25.fieldnorm_table()[ids].astype(np.uint64).sum())   # the index is written from the quantised lengths
    avg = np.float32(np.float32(total_tokens) / np.float32(max_doc))
    ranks = np.arange(1, n_ranks + 1)
    target = np.minimum(np.maximum(1, np.round(df_scale / ranks)), max_doc // 2).astype(np.int64)
    docs_l, off = [], np.zeros(n_ranks + 1, np.uint64)
    for i, df in enumerate(target):
        p = df / max_doc
        n = int(df * 1.05 + 6 * np.sqrt(df) + 16)
        d = np.cumsum(rng.geometric(p, n)) - 1
        d = d[d < max_doc].astype(np.uint32)
        docs_l.append(d)
        off[i + 1] = off[i] + d.size
    docs = np.concatenate(docs_l)
    del docs_l
    tfs = np.minimum(rng.geometric(0.6, docs.size), 255).astype(np.uint32)
    data, infos = bm25.encode_postings_csr(docs, tfs, off, ids, avg, threads=threads)
    return dict(postings=data, infos=infos, fieldnorm_ids=ids, avg=avg, n_postings=int(docs.size), off=off, total_num_tokens=total_tokens)


def log_uniform_queries(n_queries, n_terms, lo=10, hi=10_000, seed=1):
    rng = np.random.default_rng(seed)
    out = np.zeros((n_queries, n_terms), np.uint32)
    for q in range(n_queries):
        s = set()
        while len(s) < n_terms:
            s.add(int(np.exp(rng.uniform(np.log(lo), np.log(hi)))))
        out[q] = sorted(s, key=lambda _: rng.random())
    return out - 1  # rank r is term ordinal r-1


def _alg_bytes(infos, terms, docs_scored, k_out_bytes, per_doc_bytes):
    plen = np.array([infos[i].postings_len for i in range(len(infos))], np.float64)
    return float(plen[terms].sum()) + per_doc_bytes * docs_scored + k_out_bytes


def run_and(device, peaks, max_doc=10_000_000, df_scale=2.0e6, n_queries=10_000, k=1000, steps=5, warmup=3, cpu=True):
    t0 = time.perf_counter()
    ix = synth_index(max_doc, df_scale)
    gen_s = time.perf_counter() - t0
    seg = bm25.SegmentReader(ix["postings"], ix["infos"], ix["fieldnorm_ids"], device=device, total_num_tokens=ix["total_num_tokens"])
    terms = log_uniform_queries(n_queries, 2)
    top = bm25.TopDocs.with_limit(k)
    for _ in range(warmup):
        top.search_batch(seg, terms, bm25.MODE_AND)
    kms, ems, st = [], [], None
    for _ in range(steps):
        t1 = time.perf_counter()
        d, s, n, st = top.search_batch(seg, terms, bm25.MODE_AND, return_stats=True)
        ems.append((time.perf_counter() - t1) * 1e3)
        kms.append(st["kernel_ms"])
    postings = st["postings_scored"]
    kern = float(np.median(kms)); e2e = float(np.median(ems))
    alg = _alg_bytes(ix["infos"], terms, st["docs_scored"], 8.0 * float(n.sum()), 1.0)
    out = {"workload": f"{max_doc} docs, Zipf vocab (ranks<=10k materialised, {ix['n_postings']} postings), "
                       f"{n_queries} x 2-term AND, tantivy BM25, top-{k}",
           "metric": "bm25_postings_scored_per_sec", "value": postings / (kern * 1e-3), "unit": "postings/s",
           "kernel_ms_per_batch": kern, "postings_per_batch": postings, "docs_scored": st["docs_scored"],
           "blocks_decoded": st["blocks_decoded"],
           "e2e": {"value": postings / (e2e * 1e-3), "unit": "postings/s", "ms_per_batch": e2e,
                   "h2d_bytes_per_step": int(terms.size * 8 + 1024),
                   # sparse result tables cross PCIe packed (counts, then only the filled entries) when under half of the dense table is filled
                   "d2h_bytes_per_step": int(n_queries * 4 + (8 * int(n.sum()) if 2 * int(n.sum()) < n_queries * k else n_queries * k * 8))},
           "roofline": {"bound": "hbm", "kernel": "k_and3 + k_and3_select", "achieved": alg / (kern * 1e-3) / 1e9, "peak": peaks["hbm_gbs"],
                        "unit": "GB/s", "frac": alg / (kern * 1e-3) / 1e9 / peaks["hbm_gbs"], "alg_bytes_per_launch": alg},
           "index_hbm_bytes": seg.info()["hbm_bytes"], "gen_s": round(gen_s, 1), "stage_ms": seg.info()["stage_ms"]}
    if cpu:
        out["cpu_baseline"], out["parity"] = cpu_and(ix, terms, k, seg, (d, s, n))
    seg.close()
    return out


def _compare(kind, g, o, nq):
    """GPU top-k tables against the oracle's for the first nq queries: counts, doc ids and score bits."""
    gd, gs, gn = g
    od, os_, on = o
    bad = 0
    for q in range(nq):
        m = int(on[q])
        if int(gn[q]) != m or not np.array_equal(gd[q, :m], od[q, :m]) or not np.array_equal(gs[q, :m], os_[q, :m]):
            bad += 1
    return {"against": kind, "queries": int(nq), "n_mismatch": int(bad), "green": bad == 0}


def cpu_and(ix, terms, k, seg, gpu_out, sample=2048, runs=3):
    """Oracle (restated tantivy Intersection + TopNComputer, with skipping), one query per thread (dynamic schedule);
    its docs / scores for the sampled queries are compared with the GPU's (parity at full index size)."""
    import oracle
    o = oracle.Segment(ix["fieldnorm_ids"], avg_fieldnorm=ix["avg"])
    infos = ix["infos"]
    n = len(infos)
    o.set_postings(ix["postings"], [infos[i].postings_off for i in range(n)], [infos[i].postings_len for i in range(n)],
                   [infos[i].doc_freq for i in range(n)])
    t = terms[:sample]
    cache = bm25.compute_tf_cache(seg.average_fieldnorm)
    df = seg.doc_freq[t]
    uniq, inv = np.unique(df, return_inverse=True)
    w = np.array([bm25.Bm25Weight.for_one_term(int(x), seg.max_doc, seg.average_fieldnorm).weight for x in uniq], np.float32)[inv].reshape(t.shape)
    caches = np.tile(cache, (t.size, 1))
    from bench import host_threads
    threads = host_threads()
    dts = []
    for _ in range(runs):
        t0 = time.perf_counter()
        od, os_, on, _sc = o.topk_batch(t, w, caches, 0, k, threads=threads)
        dts.append(time.perf_counter() - t0)
    dt = float(np.median(dts))
    postings = int(seg.doc_freq[t].sum())
    o.close()
    par = _compare("oracle Intersection + TopNComputer on the full-size index (docs and f32 score bits)", gpu_out, (od, os_, on), t.shape[0])
    return ({"value": postings / dt, "unit": "postings/s", "cores": threads, "kind": "port", "runs_s": [round(x, 3) for x in dts],
             "sample": f"first {t.shape[0]} queries of the batch ({t.shape[0] / threads:.0f} per thread, dynamic schedule), median of {runs} runs, "
                       f"oracle Intersection + skip-list seek + TopNComputer"}, par)


def run_signal(device, peaks, max_doc=100_000_000, df_scale=2.0e7, n_queries=10_000, k=1000, steps=3, warmup=1, cpu=True):
    t0 = time.perf_counter()
    ix = synth_index(max_doc, df_scale)
    rng = np.random.default_rng(99)
    hc = rng.random(max_doc) ** 8
    rank = np.empty(max_doc, np.int64); rank[np.argsort(-hc, kind="stable")] = np.arange(max_doc)
    cols = [hc, np.maximum(10.0 - np.log(1.0 + rank.astype(np.float64)) / np.log(8.0), 0.0), rng.random(max_doc),
            1.0 / (1.0 + rng.integers(0, 1000, max_doc).astype(np.float64))]
    del rank
    coeffs = [2.0, 0.02, 2.0, 0.001]
    gen_s = time.perf_counter() - t0
    seg = bm25.SegmentReader(ix["postings"], ix["infos"], ix["fieldnorm_ids"], device=device, total_num_tokens=ix["total_num_tokens"])
    table = bm25.SignalTable(cols, device=device)
    comp = bm25.SignalComputer(seg, table, coeffs, coeff_text=0.005)
    terms = log_uniform_queries(n_queries, 5, seed=2)
    for _ in range(warmup):
        comp.top_docs_batch(terms, k)
    kms, ems, st = [], [], None
    for _ in range(steps):
        t1 = time.perf_counter()
        d, tot, n, st = comp.top_docs_batch(terms, k, return_stats=True)
        ems.append((time.perf_counter() - t1) * 1e3)
        kms.append(st["kernel_ms"])
    postings = st["postings_scored"]
    kern = float(np.median(kms)); e2e = float(np.median(ems))
    alg = _alg_bytes(ix["infos"], terms, st["docs_scored"], 12.0 * float(n.sum()), 1.0 + 8.0 * 4)
    out = {"workload": f"{max_doc} docs, Zipf vocab (ranks<=10k materialised, {ix['n_postings']} postings), {n_queries} x 5-term OR, "
                       f"Stract BM25 + 4 numeric signals (f64 linear combine), top-{k}",
           "metric": "bm25_postings_scored_per_sec", "value": postings / (kern * 1e-3), "unit": "postings/s",
           "kernel_ms_per_batch": kern, "postings_per_batch": postings, "docs_scored": st["docs_scored"],
           "e2e": {"value": postings / (e2e * 1e-3), "unit": "postings/s", "ms_per_batch": e2e,
                   "h2d_bytes_per_step": int(terms.size * 8 + 1024), "d2h_bytes_per_step": int(n_queries * k * 12 + n_queries * 4)},
           "roofline": {"bound": "hbm", "kernel": "k_or3<SIGNAL,5>", "achieved": alg / (kern * 1e-3) / 1e9, "peak": peaks["hbm_gbs"],
                        "unit": "GB/s", "frac": alg / (kern * 1e-3) / 1e9 / peaks["hbm_gbs"], "alg_bytes_per_launch": alg},
           "index_hbm_bytes": seg.info()["hbm_bytes"], "gen_s": round(gen_s, 1)}
    # production-shaped variant: Stract stops a segment after max_docs_considered candidates in doc order
    # (core/src/config/defaults.rs:38-40 = 250 000; ShortCircuitQuery, tantivy/src/query/shortcircuit.rs:100-133)
    MAXD = 250_000
    comp.top_docs_batch(terms, k, max_docs=MAXD)
    kms2 = []
    for _ in range(3):
        d2, tot2, n2, st2 = comp.top_docs_batch(terms, k, max_docs=MAXD, return_stats=True)
        kms2.append(st2["kernel_ms"])
    out["max_docs_250k"] = {"kernel_ms_per_batch": float(np.median(kms2)), "docs_scored": st2["docs_scored"],
                            "queries_per_s": n_queries / (float(np.median(kms2)) * 1e-3),
                            "note": "every query stops after its first 250 000 candidate docs (ascending doc order), then top-k of those"}
    if cpu:
        import oracle
        o = oracle.Segment(ix["fieldnorm_ids"], avg_fieldnorm=ix["avg"])
        infos = ix["infos"]; nt = len(infos)
        o.set_postings(ix["postings"], [infos[i].postings_off for i in range(nt)], [infos[i].postings_len for i in range(nt)],
                       [infos[i].doc_freq for i in range(nt)])
        from bench import host_threads
        threads = host_threads()
        t = terms[:max(16 * threads, 256)]        # >= 16 queries per thread, dynamic schedule
        cache = bm25.compute_tf_cache(seg.average_fieldnorm)
        df = seg.doc_freq[t]
        uniq, inv = np.unique(df, return_inverse=True)
        w = np.array([bm25.StractBm25Weight.for_one_term(int(x), seg.max_doc, seg.average_fieldnorm).weight for x in uniq], np.float32)[inv].reshape(t.shape)
        dts = []
        for i in range(3):
            t0 = time.perf_counter()
            od, ot, on, _sc = o.signal_topk_batch(t, w, np.tile(cache, (t.size, 1)), 1.2, 0.005, cols, coeffs, k, threads=threads)
            dts.append(time.perf_counter() - t0)
            if sum(dts) + dts[-1] > 60.0:      # bounded sample: stop repeating once a minute of CPU time is spent
                break
        dt = float(np.median(dts))
        out["cpu_baseline"] = {"value": int(seg.doc_freq[t].sum()) / dt, "unit": "postings/s", "cores": threads, "kind": "port",
                               "runs_s": [round(x, 3) for x in dts],
                               "sample": f"first {t.shape[0]} queries ({t.shape[0] / threads:.0f} per thread, dynamic schedule), median of {len(dts)} run(s), "
                                         f"oracle union + per-term seek + Stract BM25 + f64 combine + TopNComputer"}
        out["parity"] = _compare("oracle union + Stract BM25 + f64 linear combine on the full-size index (docs and f64 total bits)",
                                 (d, tot, n), (od, ot, on), t.shape[0])
        od2, ot2, on2, _sc2 = o.signal_topk_batch(t, w, np.tile(cache, (t.size, 1)), 1.2, 0.005, cols, coeffs, k, max_docs=MAXD, threads=threads)
        out["max_docs_250k"]["parity"] = _compare("oracle with the same max_docs short-circuit", (d2, tot2, n2), (od2, ot2, on2), t.shape[0])
        o.close()
    table.close(); seg.close()
    return out


def run_multi(device, peaks, max_doc=10_000_000, df_scale=2.0e6, n_queries=10_000, k=1000, steps=3, cpu=True):
    """The multi-field recall stage (SURVEY 8(f)-3) at C4 index size: three text fields of one segment (Title, CleanBody, Url),
    three query terms per field = 9 slots, signals Bm25F + Bm25Title + TitleCoverage + Bm25CleanBody + CleanBodyCoverage +
    IdfSumUrl + two numeric columns in SignalComputeOrder order; parity against the oracle restatement on sampled queries."""
    t0 = time.perf_counter()
    names = ["Title", "CleanBody", "Url"]
    ixs = [synth_index(max_doc, df_scale * f, seed=1234 + 17 * i) for i, f in enumerate((0.25, 1.0, 0.1))]
    rng = np.random.default_rng(7)
    cols = [rng.random(max_doc) ** 8, 1.0 / (1.0 + rng.integers(0, 1000, max_doc).astype(np.float64))]
    gen_s = time.perf_counter() - t0
    segs = [bm25.SegmentReader(ix["postings"], ix["infos"], ix["fieldnorm_ids"], device=device, total_num_tokens=ix["total_num_tokens"]) for ix in ixs]
    table = bm25.SignalTable(cols, device=device)
    enabled = {"Bm25F", "Bm25Title", "TitleCoverage", "Bm25CleanBody", "CleanBodyCoverage", "IdfSumUrl"}
    numeric = [("HostCentrality", 0, 2.5), ("FetchTimeMs", 1, 0.001)]
    comp = bm25.MultiFieldSignalComputer(dict(zip(names, segs)), enabled, table, numeric)
    q3 = log_uniform_queries(n_queries, 3, seed=5)
    sf = np.tile(np.repeat(np.arange(3, dtype=np.uint8), 3), (n_queries, 1))
    st = np.tile(q3, (1, 3)).astype(np.uint32)
    comp.top_docs_batch(sf, st, k)
    kms, ems, stt = [], [], None
    for _ in range(steps):
        t1 = time.perf_counter()
        d, tot, n, stt = comp.top_docs_batch(sf, st, k, return_stats=True)
        ems.append((time.perf_counter() - t1) * 1e3); kms.append(stt["kernel_ms"])
    kern = float(np.median(kms)); postings = stt["postings_scored"]
    out = {"workload": f"{max_doc} docs x 3 text fields, {n_queries} queries x 9 slots (3 terms per field), 8 signals incl. Bm25F / coverage / idf_sum, top-{k}",
           "metric": "bm25_postings_scored_per_sec", "value": postings / (kern * 1e-3), "unit": "postings/s", "kernel_ms_per_batch": kern,
           "postings_per_batch": postings, "docs_scored": stt["docs_scored"], "e2e_ms_per_batch": float(np.median(ems)), "gen_s": round(gen_s, 1)}
    if cpu:
        import oracle
        osegs = []
        for ix in ixs:
            o = oracle.Segment(ix["fieldnorm_ids"], avg_fieldnorm=ix["avg"])
            infos = ix["infos"]; nt = len(infos)
            o.set_postings(ix["postings"], [infos[i].postings_off for i in range(nt)], [infos[i].postings_len for i in range(nt)],
                           [infos[i].doc_freq for i in range(nt)])
            osegs.append(o)
        caches = comp.last_inputs["caches"]
        coefs = [np.float32(comp.field_coefficient(nm)) for nm in comp.names]
        ops = [(kind, comp.names.index(field) if field is not None else 0, chain, col, comp.coefficient(name, coef))
               for name, kind, field, chain, col, coef in comp.order.entries]
        bad, nsample = 0, 64
        t1 = time.perf_counter()
        for q in range(nsample):
            od, ot = oracle.multi_signal_topk(osegs, caches, [1.2] * 3, coefs, sf[q], st[q], comp.last_inputs["idf"][q],
                                              comp.last_inputs["idf_f"][q], ops, cols, k)
            m = int(n[q])
            bad += int(m != len(od) or not np.array_equal(d[q, :m], od) or not np.array_equal(tot[q, :m], ot))
        dt = time.perf_counter() - t1
        sample_post = int(sum(int(segs[f].doc_freq[st[q, x]]) for q in range(nsample) for x, f in enumerate(sf[q])))
        out["parity"] = {"against": "oracle multi-field restatement on the full-size fields (docs and f64 total bits)", "queries": nsample,
                         "n_mismatch": int(bad), "green": bad == 0}
        out["cpu_baseline"] = {"value": sample_post / dt, "unit": "postings/s", "cores": 1, "kind": "port",
                               "sample": f"first {nsample} queries, one thread (the oracle's multi-field path is a single-query call)"}
        for o in osegs:
            o.close()
    table.close()
    for sg in segs:
        sg.close()
    return out


def run(device, peaks, peak_src, scale=1.0, cpu=True):
    res = {"peak_source": peak_src}
    res["and_top1000_10M"] = run_and(device, peaks, max_doc=int(10_000_000 * scale), df_scale=2.0e6 * scale, cpu=cpu)
    res["or5_signals_100M"] = run_signal(device, peaks, max_doc=int(100_000_000 * scale), df_scale=2.0e7 * scale, cpu=cpu)
    try:
        res["multi_field_10M"] = run_multi(device, peaks, max_doc=int(10_000_000 * scale), df_scale=2.0e6 * scale, cpu=cpu)
    except Exception as ex:  # noqa: BLE001  (a new leg must not take the established ones down)
        res["multi_field_10M"] = {"error": repr(ex)[:300]}
    return res
