"""Times the query-plan recall path on the index of bench_bm25.run_multi (10 M docs x 3 signal fields) plus one field that is
not a signal field: the plan docset stage alone (sb200_recall_plan_docs) and the plan recall batch next to the existing union
entry point over the same slots, candidates per query for both, and docset parity on sampled queries against
tests/plan_oracle.py (posting lists read back through Docset.from_postings).  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import bench_bm25 as BB  # noqa: E402
from stract_b200 import bm25, query_plan as QP  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-doc", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=10_000)
    ap.add_argument("--k", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--sample", type=int, default=32)
    a = ap.parse_args()
    names = ["Title", "CleanBody", "Url"]
    ixs = [BB.synth_index(a.max_doc, 2.0e6 * f, seed=1234 + 17 * i) for i, f in enumerate((0.25, 1.0, 0.1, 0.01))]
    segs = [bm25.SegmentReader(ix["postings"], ix["infos"], ix["fieldnorm_ids"], total_num_tokens=ix["total_num_tokens"]) for ix in ixs]
    rng = np.random.default_rng(7)
    cols = [rng.random(a.max_doc) ** 8, 1.0 / (1.0 + rng.integers(0, 1000, a.max_doc).astype(np.float64))]
    comp = bm25.MultiFieldSignalComputer(dict(zip(names, segs[:3])), {"Bm25F", "Bm25Title", "TitleCoverage", "Bm25CleanBody", "CleanBodyCoverage", "IdfSumUrl"},
                                         bm25.SignalTable(cols), [("HostCentrality", 0, 2.5), ("FetchTimeMs", 1, 0.001)])
    nt = rng.integers(2, 5, a.queries)
    terms = BB.log_uniform_queries(a.queries, 4, seed=5)
    schema = QP.Schema(names, {"Title", "CleanBody"}, {"Title", "Url"}, set())
    qs = []
    for q in range(a.queries):
        ts = [("simple", f"t{int(x)}") for x in terms[q, :nt[q]]]
        if q % 4 == 0:
            ts.append(("site", f"t{int(terms[q, 0]) % 50}"))
        qs.append(QP.parse(ts, schema))
    fields = dict(zip(names + ["UrlForSiteOperator"], segs))
    resolve = lambda field, text: [int(text[1:])] if text[1:].isdigit() else []
    plan = QP.compile_plans(qs, fields, resolve, schema)
    sf = np.full((a.queries, 12), 0xFF, np.uint8); st = np.full((a.queries, 12), bm25.NO_TERM, np.uint32)
    for q in range(a.queries):
        for f in range(3):
            for j in range(nt[q]):
                sf[q, f * nt[q] + j] = f; st[q, f * nt[q] + j] = terms[q, j]
    docsets, pst = bm25.recall_plan_docs(plan, return_stats=True)
    dms, pms, ums = [], [], []
    for _ in range(a.steps):
        dms.append(bm25.recall_plan_docs(plan, return_stats=True)[1]["kernel_ms"])
        _, _, _, s1 = comp.top_docs_batch(sf, st, a.k, plan=plan, return_stats=True); pms.append(s1["kernel_ms"])
        _, _, _, s2 = comp.top_docs_batch(sf, st, a.k, return_stats=True); ums.append(s2["kernel_ms"])
    import plan_oracle as PLO
    post_cache = {}

    def post(s, t):
        if (s, t) not in post_cache:
            post_cache[(s, t)] = bm25.Docset.from_postings(segs[s], t).docs()
        return post_cache[(s, t)]
    bad = 0
    for q in range(0, a.queries, max(1, a.queries // a.sample)):
        lookup = [_Lazy(post, s) for s in range(4)]
        bad += int(not np.array_equal(docsets[q], np.array(PLO.program_docs(plan.programs[q], lookup), np.uint32)))
    out = {"card": card(), "max_doc": a.max_doc, "queries": a.queries, "k": a.k,
           "docset_kernel_ms": float(np.median(dms)), "plan_recall_kernel_ms": float(np.median(pms)), "union_recall_kernel_ms": float(np.median(ums)),
           "plan_candidates_per_query": pst["docs"] / a.queries, "cover_per_query": pst["cover"] / a.queries,
           "union_candidates_per_query": s2["docs_scored"] / a.queries, "groups": pst["groups"], "parity_mismatches": bad}
    print(json.dumps(out))


class _Lazy:
    def __init__(self, f, s):
        self.f, self.s = f, s

    def __getitem__(self, t):
        return self.f(self.s, t)


if __name__ == "__main__":
    main()
