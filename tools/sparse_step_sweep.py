#!/usr/bin/env python3
"""Which kernel family should run the first sparse HyperBall iteration of the benchmark graph?

Builds the graph bench.py measures (R-MAT, generated on the device), then for each forced mode -- push, frontier pull,
dense pull -- runs: reset, iterations 0 .. ITER-1 under the default policy, iteration ITER under the forced mode.  The
modes take turns, --reps times each, after one untimed round (the first forced push builds the source-major CSR).
Prints one JSON line per mode: the device ms of iteration ITER (median, min, max), its n_changed, the frontier's
out-edges and a checksum of every register after it, which must be the same for all modes.  The first line names the
card and its power limit.  Needs a GPU.

  python tools/sparse_step_sweep.py [--reps 7] [--iter 5] [--nodes N --edges E --scale S]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODES = {2: "push", 1: "frontier pull", 0: "dense pull"}


def card(index):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", str(index)],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iter", type=int, default=5, help="the iteration whose mode is forced")
    ap.add_argument("--nodes", type=int, default=25_000_000)
    ap.add_argument("--edges", type=int, default=500_000_000)
    ap.add_argument("--scale", type=int, default=25)
    ap.add_argument("--device", type=int, default=0)
    args = ap.parse_args()

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

    def forced_step(mode):
        dg.set_policy(force_mode=-1)
        dg.reset()
        for _ in range(args.iter):
            st = dg.step()
            assert st["n_changed"] > 0, "the computation converged before the forced iteration"
        dg.set_policy(force_mode=mode)
        st = dg.step()
        dg.set_policy(force_mode=-1)
        assert st["mode"] == mode, (mode, st)
        return st

    for mode in MODES:   # untimed round
        forced_step(mode)
    ms = {m: [] for m in MODES}
    last = {}
    chk = {}
    for rep in range(args.reps):
        for mode in MODES:
            st = forced_step(mode)
            ms[mode].append(st["ms"])
            last[mode] = st
            if rep == 0:
                chk[mode] = registers_checksum(dg.registers())
    for mode, name in MODES.items():
        v = ms[mode]
        print(json.dumps({"mode": mode, "family": name, "iteration": args.iter, "ms_median": round(statistics.median(v), 3),
                          "ms_min": round(min(v), 3), "ms_max": round(max(v), 3), "reps": len(v),
                          "n_changed": last[mode]["n_changed"], "frontier_out_edges": last[mode]["edges_active"],
                          "registers_checksum": chk[mode]}), flush=True)
    same = len(set(chk.values())) == 1
    print(json.dumps({"registers_equal_across_modes": same}), flush=True)
    dg.close()
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
