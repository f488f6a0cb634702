"""Times LambdaMART predict (sb200_lambdamart_predict, lambdamart.cu) on three models: the reference's shipped model
(tests/golden/lambdamart.txt, 50 trees over 29 signals) over the top 20 of 10 000 queries (200 000 documents), and seeded
synthetic models of production shape (1 000 trees x 63 leaves, 500 trees x 255 leaves) over 2e5 and 2e6 documents.
Per run: the median kernel ms over --steps calls after --warmup (CUDA events, device-resident features), the median call ms with
host features (copies included, host clock around a synchronising call), documents/s, node visits/s (visits per document counted
by the vectorised numpy restatement on a sample), model bytes on the device, parity on the sample, and the CPU rate of that numpy
restatement, labelled as such.  Prints the card and its power limit read in the same run, then one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import lambdamart_oracle as O  # noqa: E402
from stract_b200.lambdamart import LambdaMART  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30)
        return out.stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def run(name, text, thresholds, n_docs_list, steps, warmup, sample, seed):
    import torch
    model = LambdaMART.parse(text)
    om = O.Model(text)
    rng = np.random.default_rng(seed)
    base = O.random_rows(rng, min(200_000, max(n_docs_list)), thresholds)
    # parity and the CPU restatement on a sample
    S = base[:sample]
    t0 = time.perf_counter()
    want, visits = O.predict_numpy(om, S)
    cpu_s = time.perf_counter() - t0
    got = model.predict(S)
    parity = bool(np.all((np.isnan(want) & np.isnan(got)) | (got.view(np.uint64) == want.view(np.uint64))))
    out = []
    for n in n_docs_list:
        X = np.tile(base, (n // base.shape[0] + 1, 1))[:n]
        Xd = torch.from_numpy(X).cuda()
        for _ in range(warmup):
            model.predict(Xd)
            model.predict(X)
        kern, call = [], []
        for _ in range(steps):
            model.predict(Xd)
            kern.append(model.last_stats["kernel_ms"])
            t0 = time.perf_counter()
            model.predict(X)
            call.append((time.perf_counter() - t0) * 1e3)
        k_ms, c_ms = float(np.median(kern)), float(np.median(call))
        vpd = visits / sample
        r = {"workload": name, "docs": n, "trees": model.n_trees, "leaves": model.info["n_leaves"], "internal": model.info["n_internal"],
             "max_depth": model.info["max_depth"], "model_bytes": model.info["device_bytes"], "kernel_ms": round(k_ms, 4),
             "kernel_ms_min_max": [round(min(kern), 4), round(max(kern), 4)], "call_ms_host_inputs": round(c_ms, 3),
             "docs_per_s": n / (k_ms * 1e-3), "node_visits_per_doc": round(vpd, 1), "node_visits_per_s": vpd * n / (k_ms * 1e-3),
             "parity_sample_docs": sample, "parity": parity, "cpu_numpy_restatement_docs_per_s": sample / cpu_s}
        print(json.dumps(r), flush=True)
        out.append(r)
        del Xd
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=20_000)
    ap.add_argument("--small", action="store_true", help="tiny sizes: a dry run of the flow")
    a = ap.parse_args()
    c = card()
    print("card:", c, flush=True)
    big = [2_000, 5_000] if a.small else [200_000, 2_000_000]
    sample = min(a.sample, 2_000) if a.small else a.sample
    fixture = open(os.path.join(ROOT, "tests", "golden", "lambdamart.txt")).read()
    fth = sorted({n.threshold for t in O.Model(fixture).trees for n in t.nodes})
    res = run("fixture 50 trees, top 20 of 10 000 queries", fixture, fth, [2_000 if a.small else 200_000], a.steps, a.warmup, sample, 1)
    for trees, leaves, seed in [(1_000, 63, 2), (500, 255, 3)]:
        rng = np.random.default_rng(seed)
        text, th = O.random_model(rng, trees // 10 if a.small else trees, leaves)
        res += run(f"synthetic {trees} trees x {leaves} leaves", text, th, big, a.steps, a.warmup, sample, seed)
    print(json.dumps({"card": c, "results": res, "parity": all(r["parity"] for r in res)}))


if __name__ == "__main__":
    main()
