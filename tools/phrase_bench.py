"""Phrase-query benchmark (sb200_phrase_topk_batch) on the C4-shaped index, with parity against the native CPU oracle.

Index (seeded): 10 M docs, lengths LogNormal(5.5, 0.8), Zipf vocabulary with df_r = round(2e6 / r) for ranks r <= 10 000,
docs drawn through geometric gaps, tf = Geometric(0.6) capped at 255 and at the doc length -- the index of bench.py's C4 leg
-- and every posting gets tf distinct positions in [0, doc length).  Each query's phrase is then planted in a seeded share
(--plant) of its AND candidates: the next term's positions in that doc become a run starting right after the previous
term's first position.  Plants of different queries may overwrite each other; the resulting match rate is reported, and
exactness rests on the oracle comparison, not on the planting.

Batches, over one segment, top-k by (score desc, doc asc):
  phrase2          10 k 2-term phrases, ranks log-uniform in [10, 10 000], slop 0, scoring on
  phrase3          10 k 3-term phrases, slop 0, scoring on
  phrase2_noscore  the 2-term phrases, slop 0, scoring off (EnableScoring::Disabled)
  and2             the 2-term AND batch over the same term pairs (sb200_bm25_topk_batch): what verification costs
Per batch: kernel ms (the library's per-launch CUDA event time, median of --steps after --warmup) and e2e ms (the Python
call, host clock around a synchronised call), phrases / candidates / positions decoded per second, algorithmic bytes
(postings bytes of the terms + position-block bytes the candidates need + 1 B fieldnorm per candidate + 8 B x results)
over kernel time against the H100 SXM data-sheet 3.35 TB/s, the native oracle on all host threads over the first --sample
queries (median of 3) as the CPU baseline, and parity of those queries (docs and f32 score bits).  The card's name and
power limit are read in the same run.  One JSON line on stdout; exit status 1 on any parity mismatch."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from stract_b200 import bm25  # noqa: E402

HBM_GBS = 3350.0


def host_threads():
    n = os.cpu_count() or 1
    try:
        n = min(n, len(os.sched_getaffinity(0)))
    except (AttributeError, OSError):
        pass
    return max(1, n)


def synth_index(max_doc, df_scale, n_ranks=10_000, seed=1234):
    rng = np.random.default_rng(seed)
    lens = np.minimum(np.maximum(1, rng.lognormal(5.5, 0.8, max_doc)), 2e9).astype(np.uint32)
    ranks = np.arange(1, n_ranks + 1)
    target = np.minimum(np.maximum(1, np.round(df_scale / ranks)), max_doc // 2).astype(np.int64)
    docs_l, term_off = [], np.zeros(n_ranks + 1, np.uint64)
    for i, df in enumerate(target):
        n = int(df * 1.05 + 6 * np.sqrt(df) + 16)
        d = np.cumsum(rng.geometric(df / max_doc, n)) - 1
        d = d[d < max_doc].astype(np.uint32)
        docs_l.append(d)
        term_off[i + 1] = term_off[i] + d.size
    docs = np.concatenate(docs_l)
    del docs_l
    dl = lens[docs]
    tfs = np.minimum(np.minimum(rng.geometric(0.6, docs.size), 255), dl).astype(np.uint32)
    # tf distinct ascending positions per posting: sorted uniform draws in [0, len - tf] plus their rank
    pos_off = np.zeros(docs.size + 1, np.uint64)
    np.cumsum(tfs, out=pos_off[1:])
    owner = np.repeat(np.arange(docs.size, dtype=np.int64), tfs)
    span = (dl - tfs + 1).astype(np.float64)[owner]
    u = (rng.random(owner.size) * span).astype(np.uint32)
    u = u[np.lexsort((u, owner))]
    positions = (u + (np.arange(owner.size, dtype=np.int64) - pos_off[:-1][owner].astype(np.int64)).astype(np.uint32)).astype(np.uint32)
    del owner, span, u
    return {"lens": lens, "docs": docs, "term_off": term_off, "tfs": tfs, "positions": positions, "pos_off": pos_off}


def log_uniform_queries(n_queries, n_terms, seed, lo=10, hi=10_000):
    rng = np.random.default_rng(seed)
    out = np.zeros((n_queries, n_terms), np.uint32)
    for q in range(n_queries):
        s = set()
        while len(s) < n_terms:
            s.add(int(np.exp(rng.uniform(np.log(lo), np.log(hi)))))
        out[q] = sorted(s, key=lambda _: rng.random())
    return out - 1


def plant(ix, queries, share, seed):
    """Write each query's phrase into `share` of its AND candidates (see the module docstring)."""
    rng = np.random.default_rng(seed)
    docs, off, tfs, pos, poff, lens = ix["docs"], ix["term_off"], ix["tfs"], ix["positions"], ix["pos_off"], ix["lens"]
    planted = 0
    for row in queries:
        sl = [docs[int(off[t]):int(off[t + 1])] for t in row]
        common = sl[0]
        for s in sl[1:]:
            common = np.intersect1d(common, s, assume_unique=True)
        if common.size == 0:
            continue
        pick = common[rng.random(common.size) < share]
        if pick.size == 0:
            continue
        pi = [int(off[t]) + np.searchsorted(s, pick) for t, s in zip(row, sl)]
        start = pos[poff[pi[0]].astype(np.int64)].astype(np.int64)     # the first term's first position
        ok = np.ones(pick.size, bool)
        for j in range(1, len(row)):
            ok &= start + j + tfs[pi[j]].astype(np.int64) - 1 < lens[pick].astype(np.int64)
        for j in range(1, len(row)):
            p, t = pi[j][ok], tfs[pi[j][ok]].astype(np.int64)
            dst = np.repeat(poff[p].astype(np.int64), t) + (np.arange(int(t.sum())) - np.repeat(np.cumsum(t) - t, t))
            pos[dst] = (np.repeat(start[ok] + j, t) + (np.arange(int(t.sum())) - np.repeat(np.cumsum(t) - t, t))).astype(np.uint32)
        planted += int(ok.sum())
    return planted


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception:
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unknown"}


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    kms, ems, out = [], [], None
    for _ in range(steps):
        t0 = time.perf_counter()
        out = fn()
        ems.append((time.perf_counter() - t0) * 1e3)
        kms.append(out[3]["kernel_ms"])
    return out, float(np.median(kms)), float(np.median(ems))


def compare(g, o, nq):
    gd, gs, gn = g
    od, os_, on = o
    bad = 0
    for q in range(nq):
        m = int(on[q])
        if int(gn[q]) != m or not np.array_equal(gd[q, :m], od[q, :m]) or not np.array_equal(gs[q, :m].view(np.uint32), os_[q, :m].view(np.uint32)):
            bad += 1
    return {"queries": int(nq), "n_mismatch": bad, "green": bad == 0}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=10_000)
    ap.add_argument("--k", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--plant", type=float, default=0.3, help="share of each query's AND candidates that get its phrase")
    ap.add_argument("--sample", type=int, default=2048, help="queries per batch checked against the oracle (CPU baseline)")
    ap.add_argument("--no-cpu", action="store_true", help="skip the oracle (no parity, no CPU baseline)")
    a = ap.parse_args()
    from phrase_fixtures import native_batch
    t0 = time.perf_counter()
    ix = synth_index(a.docs, 2.0e6 * a.docs / 10_000_000)
    q2 = log_uniform_queries(a.queries, 2, seed=1)
    q3 = log_uniform_queries(a.queries, 3, seed=2)
    planted = plant(ix, q2, a.plant, 3) + plant(ix, q3, a.plant, 4)
    ids = bm25.fieldnorms_to_ids(ix["lens"])
    total_tokens = int(bm25.fieldnorm_table()[ids].astype(np.uint64).sum())
    avg = np.float32(np.float32(total_tokens) / np.float32(a.docs))
    data, infos = bm25.encode_postings_csr(ix["docs"], ix["tfs"], ix["term_off"], ids, avg, threads=host_threads(), record_option=2)
    pbytes, po, pl = bm25.encode_positions(ix["positions"], ix["tfs"], ix["term_off"])
    gen_s = time.perf_counter() - t0
    seg = bm25.SegmentReader(data, infos, ids, record_option=2, total_num_tokens=total_tokens, positions=pbytes, positions_ranges=(po, pl))
    plen = np.array([infos[i].postings_len for i in range(len(infos))], np.float64)
    cache = bm25.compute_tf_cache(seg.average_fieldnorm)
    csr = {"docs": ix["docs"], "term_off": ix["term_off"], "positions": ix["positions"], "pos_off": ix["pos_off"], "fieldnorm_ids": ids}
    top = bm25.TopDocs.with_limit(a.k)
    threads = host_threads()
    result = {"workload": f"{a.docs} docs, Zipf ranks <= 10 000 ({ix['docs'].size} postings, {ix['positions'].size} positions), "
                          f"{a.queries} phrases per batch, top-{a.k}, phrase planted in {a.plant:.0%} of each query's AND candidates "
                          f"({planted} plants)", "card": card(), "gen_s": round(gen_s, 1), "index_hbm_bytes": seg.info()["hbm_bytes"],
              "batches": {}}
    all_green = True
    for name, q, scoring in (("phrase2", q2, True), ("phrase3", q3, True), ("phrase2_noscore", q2, False)):
        df = seg.doc_freq[q]
        w = np.array([bm25.Bm25Weight.for_terms(r, seg.max_doc, seg.average_fieldnorm).weight for r in df], np.float32)
        offs = np.tile(np.arange(q.shape[1], dtype=np.uint32), (q.shape[0], 1))
        slops = np.zeros(q.shape[0], np.uint32)
        (d, s, n, st), kern, e2e = timed(lambda: top.search_phrase_batch(seg, q, offs, slops, scoring, weights=w, return_stats=True), a.steps, a.warmup)
        alg = float(plen[q].sum()) + st["position_bytes"] + st["candidates"] + 8.0 * float(n.sum())
        b = {"kernel_ms": kern, "e2e_ms": e2e, "phrases_per_s": q.shape[0] / (kern * 1e-3), "candidates": st["candidates"],
             "matches": st["matches"], "match_rate": st["matches"] / max(st["candidates"], 1), "results": int(n.sum()),
             "candidates_per_s": st["candidates"] / (kern * 1e-3), "positions_decoded": st["positions_decoded"],
             "positions_per_s": st["positions_decoded"] / (kern * 1e-3),
             "roofline": {"alg_bytes": alg, "achieved_gbs": alg / (kern * 1e-3) / 1e9, "peak_gbs": HBM_GBS,
                          "frac": alg / (kern * 1e-3) / 1e9 / HBM_GBS}}
        if not a.no_cpu:
            m = min(a.sample, q.shape[0])
            dts = []
            for _ in range(3):
                t1 = time.perf_counter()
                o = native_batch(csr, q[:m], offs[:m], slops[:m], w[:m], cache, scoring, a.k, threads)
                dts.append(time.perf_counter() - t1)
            dt = float(np.median(dts))
            b["cpu_baseline"] = {"phrases_per_s": m / dt, "threads": threads, "queries": m, "runs_s": [round(x, 3) for x in dts],
                                 "kind": "native oracle (tests/phrase_oracle_mt.cpp), one query per thread, median of 3"}
            b["parity"] = compare((d, s, n), o, m)
            all_green &= b["parity"]["green"]
        result["batches"][name] = b
    (d, s, n, st), kern, e2e = timed(lambda: top.search_batch(seg, q2, bm25.MODE_AND, return_stats=True), a.steps, a.warmup)
    alg = float(plen[q2].sum()) + st["docs_scored"] + 8.0 * float(n.sum())
    result["batches"]["and2"] = {"kernel_ms": kern, "e2e_ms": e2e, "queries_per_s": q2.shape[0] / (kern * 1e-3),
                                 "docs_scored": st["docs_scored"],
                                 "roofline": {"alg_bytes": alg, "achieved_gbs": alg / (kern * 1e-3) / 1e9, "peak_gbs": HBM_GBS,
                                              "frac": alg / (kern * 1e-3) / 1e9 / HBM_GBS}}
    result["batches"]["phrase2"]["kernel_ms_over_and2"] = result["batches"]["phrase2"]["kernel_ms"] / kern
    result["parity_green"] = bool(all_green) if not a.no_cpu else None
    seg.close()
    print(json.dumps(result))
    return 0 if (a.no_cpu or all_green) else 1


if __name__ == "__main__":
    sys.exit(main())
