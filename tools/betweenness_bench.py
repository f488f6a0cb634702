"""Times betweenness centrality (sb200_betweenness, graph_betweenness.cu) on the C1 graph (synth.uniform_graph(100 000,
1 000 000, seed=42), every link counted) with every node as a source, in ascending id order -- exactly the reference's
100 000-source cap.  Reports the call time on the device (CUDA events around the synchronising call: staging of the
id-ordered out-rows, every level's kernels and its host round trip, the output copy), source x edge visits per second, the
canonical-order CPU restatement (tests/betweenness_oracle_mt.cpp) on all host cores over the same workload, and parity of
every node's f64 centrality and of max_dist.  Prints the card and its power limit read in the same run, then one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import betweenness_oracle as B  # noqa: E402
from stract_b200 import synth  # noqa: E402
from stract_b200.webgraph import DeviceGraph, Webgraph  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30)
        return out.stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=100_000)
    ap.add_argument("--edges", type=int, default=1_000_000)
    ap.add_argument("--sources", type=int, default=100_000)
    ap.add_argument("--no-cpu", action="store_true", help="skip the CPU restatement (and the parity check)")
    args = ap.parse_args()
    import torch
    c = card()
    print("card:", c, flush=True)
    d = synth.uniform_graph(args.nodes, args.edges, seed=42)
    a = (d["from_lo"], d["from_hi"], d["to_lo"], d["to_hi"], d["rel_flags"])
    ids_lo, ids_hi, fr, tr = B.rank_links(*a[:4])
    n = len(ids_lo)
    src = np.arange(min(args.sources, n), dtype=np.uint32)
    ids = [(int(ids_hi[s]) << 64) | int(ids_lo[s]) for s in src]
    kept = int(np.unique((fr.astype(np.uint64) << np.uint64(32) | tr)[fr != tr]).size)
    dg = DeviceGraph(Webgraph.from_arrays(*a), skipped_rel=0)
    try:
        dg.betweenness(ids[:640])   # warm-up: modules loaded, adjacency path exercised
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        lo, hi, cent, md = dg.betweenness(ids)
        e1.record()
        torch.cuda.synchronize()
        gpu_ms = e0.elapsed_time(e1)
    finally:
        dg.close()
    print(f"gpu: {gpu_ms:.1f} ms for {len(src)} sources", flush=True)
    r = {"graph": f"C1 uniform {args.nodes} x {args.edges} seed 42", "nodes": n, "kept_edges": kept, "sources": len(src),
         "gpu_call_ms": round(gpu_ms, 1), "gpu_source_edge_visits_per_s": len(src) * kept / (gpu_ms / 1e3), "max_dist": md,
         "entries": len(cent)}
    if not args.no_cpu:
        threads = os.cpu_count() or 1
        t0 = time.perf_counter()
        oc, reached, omd = B.canonical(n, fr, tr, src, threads=threads, chunk=2000,
                                       progress=lambda k: print(f"cpu oracle: {k} sources, {time.perf_counter() - t0:.0f} s", flush=True))
        cpu_s = time.perf_counter() - t0
        keys = np.flatnonzero(reached)
        parity = bool(np.array_equal(lo, ids_lo[keys]) and np.array_equal(hi, ids_hi[keys]) and B.same_bits(cent, oc[keys]))
        r.update({"cpu_oracle_s": round(cpu_s, 2), "cpu_threads": threads, "cpu_source_edge_visits_per_s": len(src) * kept / cpu_s,
                  "speedup_vs_cpu_oracle": round(cpu_s * 1e3 / gpu_ms, 1), "parity_centrality": parity, "parity_max_dist": md == omd})
    print(json.dumps({"card": c, "result": r}))


if __name__ == "__main__":
    main()
