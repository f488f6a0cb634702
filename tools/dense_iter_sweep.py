#!/usr/bin/env python3
"""How large should the persisting L2 window and the L1 budget of the hub rows be for the dense HyperBall iterations?

Builds the graph bench.py measures (R-MAT, generated on the device), then for each pair of a window size (the handle
option "l2_window_mb") and an L1 hub budget (the handle option "l1_hub_kb"; L1 and L2 residency interact, so every pair
of the two lists is run) runs whole centrality computations (run() after a reset) with the per-kernel profile on.  The
settings take turns, --reps times each, after one untimed round.  Prints one JSON line per setting: the device ms of run()
(median, min, max), the median ms of every iteration, the per-kernel ms per computation (sb200_hyperball_get_profile), the
changed count of every iteration and a checksum of every register after the last one; the last two must be the same for
all settings.  The first line names the card, its power limit and its max SM clock (read only).  Needs a GPU.

  python tools/dense_iter_sweep.py [--window-mb 16,20,24,28,32] [--l1-hub-kb 0,128,1048576] [--reps 5] [--nodes N --edges E --scale S]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card(index):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", str(index)],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-mb", default="16,20,24,28,32", help="comma-separated window sizes in MiB (0: no window)")
    ap.add_argument("--l1-hub-kb", default="1048576", help="comma-separated L1 hub budgets in KiB (0: no gather through L1; the "
                    "default, more than the 64 B rows of C2's 14.4 M nodes: every gather through L1, as the handle's default)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--nodes", type=int, default=25_000_000)
    ap.add_argument("--edges", type=int, default=500_000_000)
    ap.add_argument("--scale", type=int, default=25)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()
    variants = [(float(w), float(k)) for w in args.window_mb.split(",") if w.strip()
                for k in args.l1_hub_kb.split(",") if k.strip()]

    import torch
    from bench import gen_device_graph, registers_checksum
    from stract_b200 import lib
    from stract_b200.webgraph import DeviceGraph, Webgraph

    assert torch.cuda.is_available(), "the sweep needs a GPU"
    torch.cuda.set_device(args.device)
    print(json.dumps({"card": torch.cuda.get_device_name(args.device), "nvidia_smi": card(args.device)}), flush=True)
    cols = gen_device_graph(torch, lib(), args.device, args.nodes, args.edges, args.scale)
    torch.cuda.synchronize()
    dg = DeviceGraph(Webgraph.from_arrays(*cols), device=args.device)
    del cols
    torch.cuda.empty_cache()
    info = dg.info()
    print(json.dumps({"n_nodes": info["n_nodes"], "kept_edges": info["n_edges_kept"]}), flush=True)

    def computation(v):
        dg.set_option("l2_window_mb", v[0])
        dg.set_option("l1_hub_kb", v[1])
        dg.reset()
        dg.set_profiling(True)
        iters, stats = dg.run()
        prof = dg.profile()
        dg.set_profiling(False)
        return dg.last_run_ms(), stats, prof

    for v in variants:   # untimed round
        computation(v)
    runs = {v: [] for v in variants}
    chk, changed = {}, {}
    for rep in range(args.reps):
        for v in variants:
            ms, stats, prof = computation(v)
            runs[v].append((ms, stats, prof))
            if rep == 0:
                chk[v] = registers_checksum(dg.registers())
                changed[v] = [s["n_changed"] for s in stats]
    for v in variants:
        r = runs[v]
        tot = [x[0] for x in r]
        n_it = len(r[0][1])
        per_iter = [round(statistics.median(x[1][t]["ms"] for x in r), 3) for t in range(n_it)]
        kernels = {}
        for p in r[0][2]:
            if p["launches"]:
                kernels[p["name"]] = round(statistics.median(next(q["ms"] for q in x[2] if q["name"] == p["name"]) for x in r), 3)
        print(json.dumps({"window_mb": v[0], "l1_hub_kb": v[1], "ms_median": round(statistics.median(tot), 3), "ms_min": round(min(tot), 3),
                          "ms_max": round(max(tot), 3), "reps": len(tot), "per_iter_ms_median": per_iter,
                          "modes": [s["mode"] for s in r[0][1]], "kernel_ms_median": kernels,
                          "n_changed": changed[v], "registers_checksum": chk[v]}), flush=True)
    same = len({json.dumps([changed[v], chk[v]]) for v in variants}) == 1
    print(json.dumps({"results_equal_across_settings": same}), flush=True)
    dg.close()
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
