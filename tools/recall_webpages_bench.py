"""Times the recall webpages (sb200_multi_signal_webpages) on a 10 M-doc index: Title and CleanBody with positions (record
option 2), Url without, 10 000 queries of 2-4 terms, each query's top-20 and top-200 from the plan recall batch as the documents.
Reports the median kernel ms over --steps runs after --warmup, documents/s, positions decoded/s, algorithmic bytes over kernel
time against 3.35 TB/s (DESIGN.md §3, "Recall webpages"), parity against tests/webpage_oracle.py on sampled queries and the
CPU rate of that Python restatement on them.  Prints the card and its power limit read in the same run, then one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from stract_b200 import bm25, query_plan as QP  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def synth_field(max_doc, df_scale, seed, positions, n_ranks=10_000):
    """bench_bm25.synth_index's Zipf posting lists, kept as CSR (docs, tfs, positions) so the oracle can read them back"""
    rng = np.random.default_rng(seed)
    lens = np.minimum(np.maximum(1, rng.lognormal(5.5, 0.8, max_doc)), 2e9).astype(np.uint32)
    ids = bm25.fieldnorms_to_ids(lens)
    total = int(bm25.fieldnorm_table()[ids].astype(np.uint64).sum())
    avg = np.float32(np.float32(total) / np.float32(max_doc))
    target = np.minimum(np.maximum(1, np.round(df_scale / np.arange(1, n_ranks + 1))), max_doc // 2).astype(np.int64)
    docs_l, off = [], np.zeros(n_ranks + 1, np.uint64)
    for i, df in enumerate(target):
        n = int(df * 1.05 + 6 * np.sqrt(df) + 16)
        d = np.cumsum(rng.geometric(df / max_doc, n)) - 1
        d = d[d < max_doc].astype(np.uint32)
        docs_l.append(d)
        off[i + 1] = off[i] + d.size
    docs = np.concatenate(docs_l)
    tfs = np.minimum(rng.geometric(0.6, docs.size), 255).astype(np.uint32)
    data, infos = bm25.encode_postings_csr(docs, tfs, off, ids, avg, threads=16, record_option=2 if positions else 1)
    f = dict(docs=docs, tfs=tfs, off=off, ids=ids)
    if positions:   # ascending positions per posting: cumulative gaps restarted at every posting
        gaps = rng.integers(1, 24, int(tfs.sum())).astype(np.uint64)
        cs = np.cumsum(gaps)
        pstart = np.zeros(tfs.size, np.int64)
        pstart[1:] = np.cumsum(tfs.astype(np.int64))[:-1]
        base = np.where(pstart > 0, cs[np.maximum(pstart, 1) - 1], 0)
        pos = (cs - np.repeat(base, tfs)).astype(np.uint32)
        pdata, po, pl = bm25.encode_positions(pos, tfs, off)
        seg = bm25.SegmentReader(data, infos, ids, record_option=2, total_num_tokens=total, positions=pdata, positions_ranges=(po, pl))
        f.update(pos=pos, pstart=pstart)
    else:
        seg = bm25.SegmentReader(data, infos, ids, total_num_tokens=total)
    f.update(seg=seg, plen=np.array([infos[i].postings_len for i in range(len(infos))], np.float64))
    return f


def oracle_field(f, needed):
    """the oracle's view of a field, restricted to the terms the sampled queries use"""
    terms = []
    for t in range(f["off"].size - 1):
        if t not in needed:
            terms.append({"docs": [], "tfs": []})
            continue
        a, b = int(f["off"][t]), int(f["off"][t + 1])
        if "pos" in f:
            terms.append({"docs": f["docs"][a:b], "positions": [f["pos"][int(f["pstart"][p]):int(f["pstart"][p]) + int(f["tfs"][p])] for p in range(a, b)]})
        else:
            terms.append({"docs": f["docs"][a:b], "tfs": f["tfs"][a:b]})
    return {"terms": terms, "ids": f["ids"]}


def alg_bytes(fields, sf, st, docs, n, n_ops, n_cols, pos_bytes):
    """per (query, slot): the distinct 128-posting blocks its sorted documents fall in, at the term's mean block size; per document:
    a fieldnorm byte per field, the signal row, and the outputs (2 x n_ops f64, the boost, 2 u32 slops); the position bytes decoded"""
    total = 0.0
    for q in range(sf.shape[0]):
        d = np.sort(docs[q, :n[q]])
        for x in range(sf.shape[1]):
            if sf[q, x] == 0xFF:
                continue
            f = fields[int(sf[q, x])]; t = int(st[q, x])
            a, b = int(f["off"][t]), int(f["off"][t + 1])
            nblk = max(1, (b - a + 127) // 128)
            blocks = np.unique(np.minimum(np.searchsorted(f["docs"][a:b], d) // 128, nblk - 1)).size
            total += blocks * f["plen"][t] / nblk
    nd = float(n.sum())
    return total + nd * (len(fields) + 8 * n_cols + 16 * n_ops + 16) + pos_bytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-doc", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=10_000)
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=16)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    names = ["Title", "CleanBody", "Url"]
    fields = [synth_field(a.max_doc, 2.0e6 * s * a.max_doc / 1e7, 1234 + 17 * i, positions=i < 2) for i, s in enumerate((0.25, 1.0, 0.1))]
    rng = np.random.default_rng(7)
    cols = [rng.random(a.max_doc) ** 8]
    comp = bm25.MultiFieldSignalComputer(dict(zip(names, [f["seg"] for f in fields])),
                                         {"Bm25F", "Bm25Title", "TitleCoverage", "Bm25CleanBody", "CleanBodyCoverage", "IdfSumUrl"},
                                         bm25.SignalTable(cols), [("HostCentrality", 0, 2.0)])
    nt = rng.integers(2, 5, a.queries)
    terms = np.zeros((a.queries, 4), np.uint32)
    for q in range(a.queries):
        terms[q] = rng.permutation(np.unique(np.exp(rng.uniform(np.log(10), np.log(10_000), 12)).astype(np.int64) - 1))[:4]
    schema = QP.Schema(names, {"Title", "CleanBody"}, {"Title", "Url"}, set())
    qs = [QP.parse([("simple", f"t{int(x)}") for x in terms[q, :nt[q]]], schema) for q in range(a.queries)]
    plan = QP.compile_plans(qs, dict(zip(names, [f["seg"] for f in fields])), lambda field, text: [int(text[1:])] if text[1:].isdigit() else [], schema)
    sf = np.full((a.queries, 12), 0xFF, np.uint8); st = np.full((a.queries, 12), bm25.NO_TERM, np.uint32)
    for q in range(a.queries):
        for f in range(3):
            for j in range(nt[q]):
                sf[q, f * nt[q] + j] = f; st[q, f * nt[q] + j] = terms[q, j]
    out = {"card": card(), "max_doc": a.max_doc, "queries": a.queries}
    for k in (20, 200):
        docs, totals, n = comp.top_docs_batch(sf, st, k, plan=plan)
        for _ in range(a.warmup):
            comp.ranking_webpages(sf, st, docs, n)
        kms, stats = [], None
        for _ in range(a.steps):
            wp, stats = comp.ranking_webpages(sf, st, docs, n, return_stats=True)
            kms.append(stats["kernel_ms"])
        ms = float(np.median(kms))
        nb = alg_bytes(fields, sf, st, docs, n, len(comp.order.entries), len(cols), stats["position_bytes"])
        # parity on sampled queries, and the CPU rate of the Python restatement on them
        import webpage_oracle as WO
        have = np.flatnonzero(n > 0)
        sample = have[::max(1, have.size // a.sample)][:a.sample].tolist()
        needed = [set() for _ in names]
        for q in sample:
            for x in range(12):
                if sf[q, x] != 0xFF:
                    needed[int(sf[q, x])].add(int(st[q, x]))
        ops = [(kind, names.index(field) if field is not None else 0, chain, col, comp.coefficient(nm, coef))
               for nm, kind, field, chain, col, coef in comp.order.entries]
        O = WO.Oracle([oracle_field(f, nd) for f, nd in zip(fields, needed)], comp.last_inputs["caches"], comp.k1,
                      [np.float32(comp.field_coefficient(nm)) for nm in names], ops, cols)
        bad, n_cpu, t0 = 0, 0, time.perf_counter()
        for q in sample:
            xs = [x for x in range(12) if sf[q, x] != 0xFF]
            slots = [(int(sf[q, x]), int(st[q, x])) for x in xs]
            idf = [comp.last_inputs["idf"][q][x] for x in xs]; idf_f = [comp.last_inputs["idf_f"][q][x] for x in xs]
            for i in range(int(n[q])):
                v, s, b, sl = O.page(int(docs[q, i]), slots, idf, idf_f, dist=(0, 1))
                ok = np.array_equal(np.asarray(wp.scores[q, i]).view(np.uint64), np.asarray(s, np.float64).view(np.uint64))
                ok = ok and float(wp.boosts[q, i]) == b and tuple(int(y) for y in wp.min_slop[q, i]) == sl
                ok = ok and O.total(wp.scores[q, i], wp.boosts[q, i]) == float(totals[q, i])
                bad += int(not ok); n_cpu += 1
        cpu_s = time.perf_counter() - t0
        out[f"top{k}"] = {"docs": stats["docs"], "kernel_ms": ms, "kernel_ms_all": kms, "ms": stats["ms"],
                          "docs_per_s": stats["docs"] / (ms * 1e-3), "docs_with_positions": stats["docs_with_positions"],
                          "positions_decoded": stats["positions_decoded"], "positions_per_s": stats["positions_decoded"] / (ms * 1e-3),
                          "alg_bytes": nb, "alg_bytes_per_s": nb / (ms * 1e-3), "hbm_share": nb / (ms * 1e-3) / HBM_BYTES_PER_S,
                          "parity_docs": n_cpu, "parity_mismatches": bad,
                          "cpu_python_restatement_docs_per_s": n_cpu / cpu_s if cpu_s > 0 else None}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
