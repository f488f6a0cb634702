"""Timing of kernel switches on one resident index (`python tools/bm25_variants.py and|signal [scale]`): the AND occupancy
variants need a fresh process each (static switch), the union kernel's TMA staging toggles per call."""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import bench_bm25  # noqa: E402
from stract_b200 import bm25  # noqa: E402

what = sys.argv[1]
if what == "and":
    ix = bench_bm25.synth_index(10_000_000, 2.0e6)
    seg = bm25.SegmentReader(ix["postings"], ix["infos"], ix["fieldnorm_ids"], total_num_tokens=ix["total_num_tokens"])
    terms = bench_bm25.log_uniform_queries(10_000, 2)
    top = bm25.TopDocs.with_limit(1000)
    for _ in range(3):
        top.search_batch(seg, terms, bm25.MODE_AND)
    ks, es = [], []
    for _ in range(7):
        t0 = time.perf_counter()
        d, s, n, st = top.search_batch(seg, terms, bm25.MODE_AND, return_stats=True)
        es.append((time.perf_counter() - t0) * 1e3); ks.append(st["kernel_ms"])
    print("AND occ", os.environ.get("SB200_AND3_OCC", "5"), "kernel_ms", round(float(np.median(ks)), 3), "call_ms(device)", round(st["ms"], 3),
          "e2e_ms", round(float(np.median(es)), 3), "checksum", int(d.astype(np.uint64).sum()), int(n.sum()))
else:
    scale = float(sys.argv[2]) if len(sys.argv) > 2 else 1.0
    max_doc = int(100_000_000 * scale)
    ix = bench_bm25.synth_index(max_doc, 2.0e7 * scale)
    rng = np.random.default_rng(99)
    cols = [rng.random(max_doc) ** 8, rng.random(max_doc), rng.random(max_doc), 1.0 / (1.0 + rng.integers(0, 1000, max_doc).astype(np.float64))]
    seg = bm25.SegmentReader(ix["postings"], ix["infos"], ix["fieldnorm_ids"], total_num_tokens=ix["total_num_tokens"])
    comp = bm25.SignalComputer(seg, bm25.SignalTable(cols), [2.0, 0.02, 2.0, 0.001], coeff_text=0.005)
    terms = bench_bm25.log_uniform_queries(10_000, 5, seed=2)
    ref = None
    for tma in ("1", "0", "1", "0"):
        os.environ["SB200_BM25_TMA"] = tma
        comp.top_docs_batch(terms, 1000)
        ks = []
        for _ in range(2):
            d, tot, n, st = comp.top_docs_batch(terms, 1000, return_stats=True)
            ks.append(st["kernel_ms"])
        same = None if ref is None else bool(np.array_equal(d, ref[0]) and np.array_equal(tot, ref[1]))
        if ref is None:
            ref = (d.copy(), tot.copy())
        print("SIGNAL tma", tma, "kernel_ms", [round(x, 2) for x in ks], "identical to first", same, flush=True)
    # tantivy OR (5 terms) on the same index, both settings
    top = bm25.TopDocs.with_limit(1000)
    for tma in ("1", "0"):
        os.environ["SB200_BM25_TMA"] = tma
        top.search_batch(seg, terms[:2000], bm25.MODE_OR)
        d, s, n, st = top.search_batch(seg, terms[:2000], bm25.MODE_OR, return_stats=True)
        print("OR5 (2000 queries) tma", tma, "kernel_ms", round(st["kernel_ms"], 2), flush=True)
