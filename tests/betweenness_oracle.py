"""Betweenness oracles and fixtures (no pytest).

- `literal`: a line-by-line transcription of the reference's `calculate` (crates/core/src/webgraph/centrality/betweenness.rs:29-146):
  FIFO queue, visit stack, predecessor lists, i32 sigma wrapping like the release build, the dependency update in reverse
  visit order.  The reference's forward links come in the store's order; here they come in ascending node id.
- `canonical`: the threaded C++ restatement (betweenness_oracle_mt.cpp) in the order this project pins: delta[v] sums over v's
  successors in ascending node id, centrality[w] sums the per-source deltas in source order.  The device is compared with
  it bit for bit.
Nodes are dense ranks 0..n-1 (ascending id); edges are (from_rank, to_rank) pairs.
"""
import ctypes as C
import os
import subprocess
import tempfile
from collections import deque

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def _i32(x):
    return ((x + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def literal(n, fr, tr, sources):
    """(centrality {rank: f64}, max_dist) exactly as the reference computes them for this source order and link order."""
    out = [[] for _ in range(n)]
    for a, b in sorted(set((int(a), int(b)) for a, b in zip(fr, tr))):
        out[a].append(b)          # a self-loop stays: the reference's loop does nothing with it
    centrality = {}
    max_dist = 0
    cnt = 0
    for s in sources:
        s = int(s)
        cnt += 1
        centrality.setdefault(s, 0.0)
        stack, pred, sigma, dist = [], {}, {s: 1}, {s: 0}
        q = deque([s])
        while q:
            v = q.popleft()
            stack.append(v)
            for w in out[v]:
                if w not in dist:
                    q.append(w)
                    dist[w] = dist[v] + 1
                if dist[w] == dist[v] + 1:
                    sigma[w] = _i32(sigma.get(w, 0) + sigma.get(v, 0))
                    pred.setdefault(w, []).append(v)
        max_dist = max(max_dist, max(dist.values()))
        delta = {}
        while stack:
            w = stack.pop()
            for v in pred.get(w, []):
                dv = delta.get(v, 0.0)
                delta[v] = dv + _fdiv(float(sigma[v]), float(sigma[w])) * (1.0 + delta.get(w, 0.0))
            if w != s:
                centrality[w] = centrality.get(w, 0.0) + delta.get(w, 0.0)
    norm = float(cnt) * (float(cnt) - 1.0)
    return {k: _fdiv(v, norm) for k, v in centrality.items()}, max_dist


def _fdiv(a, b):
    """IEEE f64 a / b (Python raises on a zero divisor; Rust and C do not)."""
    if b != 0.0:
        return a / b
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.float64(a) / np.float64(b))


_NATIVE = None


def _native():
    global _NATIVE
    if _NATIVE is None:
        out = os.path.join(tempfile.mkdtemp(prefix="bc_oracle_"), "libbc_oracle.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-pthread",
                               os.path.join(HERE, "betweenness_oracle_mt.cpp"), "-o", out])
        L = C.CDLL(out)
        L.bc_oracle.restype = C.c_int
        _NATIVE = L
    return _NATIVE


def canonical(n, fr, tr, sources, threads=None, chunk=None, progress=None):
    """(centrality f64 [n], reached bool [n], max_dist): the canonical-order restatement; `reached` is the output key set.
    With `chunk`, the sources go to the native code `chunk` at a time (the sums continue in source order) and
    `progress(done)` is called after each."""
    fr = np.ascontiguousarray(fr, np.uint32); tr = np.ascontiguousarray(tr, np.uint32)
    src = np.ascontiguousarray(sources, np.uint32)
    cent = np.zeros(max(n, 1), np.float64); reached = np.zeros(max(n, 1), np.uint8); md = C.c_int32(0)
    P = lambda a: C.c_void_p(a.ctypes.data)
    step = chunk or max(src.size, 1)
    for a in range(0, src.size, step):
        part = np.ascontiguousarray(src[a:a + step])
        rc = _native().bc_oracle(C.c_uint32(n), P(fr), P(tr), C.c_uint64(fr.size), P(part), C.c_uint32(part.size),
                                 C.c_int(threads or os.cpu_count() or 1), P(cent), P(reached), C.byref(md))
        assert rc == 0, "source rank out of range"
        if progress:
            progress(a + part.size)
    k = float(src.size)
    with np.errstate(divide="ignore", invalid="ignore"):
        cent = cent / np.float64(k * (k - 1.0))      # n == 1 divides by zero like the reference
    return cent[:n], reached[:n].astype(bool), md.value


def as_map(cent, reached):
    return {int(v): float(cent[v]) for v in np.flatnonzero(reached)}


def same_bits(a, b):
    """f64 arrays equal bit for bit; a NaN equals any NaN (x86 and the GPU give 0/0 different payloads)."""
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    if a.shape != b.shape:
        return False
    nan = np.isnan(a)
    return bool(np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan].view(np.uint64), b[~nan].view(np.uint64)))


# ---- graphs (rank form) ------------------------------------------------------------------------------------------------

def path(k):
    """0 -> 1 -> ... -> k-1: the reference's `create_path_graph`."""
    return k, np.arange(k - 1, dtype=np.uint32), np.arange(1, k, dtype=np.uint32)


def diamonds(k):
    """A chain of k diamonds m_i -> {a_i, b_i} -> m_{i+1}: 2^k shortest paths from m_0 to m_k (the i32 sigma wraps to
    -2^31 at k = 31 and to 0 at k = 32).  Node ranks: m_i = 3i, a_i = 3i + 1, b_i = 3i + 2."""
    fr, tr = [], []
    for i in range(k):
        m, a, b, m2 = 3 * i, 3 * i + 1, 3 * i + 2, 3 * i + 3
        fr += [m, m, a, b]; tr += [a, b, m2, m2]
    return 3 * k + 1, np.array(fr, np.uint32), np.array(tr, np.uint32)


def random_graph(n, m, seed, self_loops=True):
    rng = np.random.default_rng(seed)
    fr = rng.integers(0, n, m).astype(np.uint32); tr = rng.integers(0, n, m).astype(np.uint32)
    if not self_loops:
        keep = fr != tr
        fr, tr = fr[keep], tr[keep]
    return n, fr, tr


def random_tree(n, seed):
    """Every node but 0 has one parent: from any source, every node has at most one successor on the shortest-path DAG."""
    rng = np.random.default_rng(seed)
    child = np.arange(1, n, dtype=np.uint32)
    parent = np.array([rng.integers(0, c) for c in child], np.uint32)
    return n, parent, child


def to_ids(n, seed=0):
    """Ascending u128 node ids for ranks 0..n-1 (some with a high word) -> (lo, hi) uint64 arrays."""
    rng = np.random.default_rng(seed)
    ids = sorted(set(int(x) for x in rng.integers(1, 1 << 62, 3 * n + 8)))[:n]
    ids = [(x << 64 | x * 7) if i % 3 == 0 else x for i, x in enumerate(ids)]
    ids.sort()
    return np.array([x & (2**64 - 1) for x in ids], np.uint64), np.array([x >> 64 for x in ids], np.uint64), ids


def edge_arrays(n, fr, tr, rel=None, seed=0):
    """(from_lo, from_hi, to_lo, to_hi, rel_flags) of a rank-form graph over `to_ids(n, seed)`, plus the id list."""
    lo, hi, ids = to_ids(n, seed)
    fr = np.asarray(fr, np.int64); tr = np.asarray(tr, np.int64)
    rel = np.zeros(fr.size, np.uint64) if rel is None else np.asarray(rel, np.uint64)
    return (lo[fr].copy(), hi[fr].copy(), lo[tr].copy(), hi[tr].copy(), rel), ids


def rank_links(from_lo, from_hi, to_lo, to_hi):
    """(ids_lo, ids_hi, from_rank, to_rank) of an id-form edge stream (every link; numpy, any size)."""
    k = np.concatenate([np.stack([np.asarray(from_hi, np.uint64), np.asarray(from_lo, np.uint64)], 1),
                        np.stack([np.asarray(to_hi, np.uint64), np.asarray(to_lo, np.uint64)], 1)])
    ids, inv = np.unique(k, axis=0, return_inverse=True)
    inv = inv.reshape(-1).astype(np.uint32)
    m = len(from_lo)
    return ids[:, 1].copy(), ids[:, 0].copy(), inv[:m], inv[m:]
