"""ctypes binding of the CPU oracle (oracle/liboracle.so).  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

# SKIPPED_REL of crates/core/src/webgraph/centrality/harmonic.rs:36-49 over the bit positions of
# crates/core/src/webpage/html/links.rs:114-141
SKIPPED_REL_MASK = sum(1 << b for b in (8, 10, 11, 13, 14, 15, 16, 17, 18, 19, 21, 22))


def build(force=False):
    so = os.path.join(_HERE, "liboracle.so")
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".cpp", ".h"))]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "liboracle.so"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _proto(_LIB)
    return _LIB


_u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
_u32p = np.ctypeslib.ndpointer(np.uint32, flags="C_CONTIGUOUS")
_u64p = np.ctypeslib.ndpointer(np.uint64, flags="C_CONTIGUOUS")
_f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
_f64p = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")


def _proto(L):
    def f(name, res, *args):
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = list(args)

    f("orc_hll_add", None, _u8p, C.c_int, C.c_uint64)
    f("orc_hll_add_range", None, _u8p, C.c_int, C.c_uint64, C.c_uint64)
    f("orc_hll_merge", None, _u8p, _u8p, C.c_int)
    f("orc_hll_size", C.c_uint64, _u8p, C.c_int)
    f("orc_hll64_linear_counting", C.c_double, C.c_uint32)
    f("orc_kahan_add", None, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_double)
    f("orc_bloom_num_bits", C.c_uint64, C.c_uint64, C.c_double)
    f("orc_bloom_new", C.c_void_p, C.c_uint64, C.c_double)
    f("orc_bloom_free", None, C.c_void_p)
    f("orc_bloom_insert", None, C.c_void_p, C.c_uint64)
    f("orc_bloom_contains", C.c_int, C.c_void_p, C.c_uint64)
    f("orc_bloom_estimate_card", C.c_uint64, C.c_void_p)
    edge_args = (_u64p, _u64p, _u64p, _u64p, _u64p, C.c_uint64, C.c_uint64)
    f("orc_hb_faithful_run", C.c_void_p, *edge_args, C.c_uint32)
    f("orc_hb_faithful_num_nodes", C.c_uint64, C.c_void_p)
    f("orc_hb_faithful_iters", C.c_uint32, C.c_void_p)
    f("orc_hb_faithful_len", C.c_uint64, C.c_void_p)
    f("orc_hb_faithful_result", None, C.c_void_p, _u64p, _u64p, _f64p)
    f("orc_hb_faithful_free", None, C.c_void_p)
    f("orc_hb_dense_create", C.c_void_p, *edge_args, C.c_int)
    f("orc_hb_dense_num_nodes", C.c_uint64, C.c_void_p)
    f("orc_hb_dense_num_edges", C.c_uint64, C.c_void_p)
    f("orc_hb_dense_iters", C.c_uint64, C.c_void_p)
    f("orc_hb_dense_step", C.c_uint64, C.c_void_p)
    f("orc_hb_dense_run", C.c_uint32, C.c_void_p, C.c_uint32)
    f("orc_hb_dense_registers", None, C.c_void_p, C.c_uint64, C.c_uint64, _u8p)
    f("orc_hb_dense_ids", None, C.c_void_p, _u64p, _u64p)
    f("orc_hb_dense_kahan", None, C.c_void_p, _f64p, _f64p)
    f("orc_hb_dense_result", C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p)
    f("orc_hb_dense_free", None, C.c_void_p)
    f("orc_hb_dense_create_mt", C.c_void_p, *edge_args, C.c_int)
    f("orc_hb_dense_reset", None, C.c_void_p)
    f("orc_hb_dense_num_self_loops", C.c_uint64, C.c_void_p)
    f("orc_hb_dense_registers_ptr", C.c_void_p, C.c_void_p)
    f("orc_graph_distances", None, C.c_uint32, _u32p, _u32p, C.c_uint64, _u32p, _u32p, C.c_uint32, C.c_uint32, C.c_int, C.c_int, _u8p)
    f("orc_inbound_similarity", None, C.c_uint32, _u64p, _u64p, _u32p, _u32p, C.c_uint64, _u32p, C.c_uint32, _u32p, C.c_uint32, _u32p, C.c_uint32,
      C.c_int, C.c_double, _f64p)
    f("orc_approx_harmonic", None, C.c_uint32, _u32p, _u32p, C.c_uint64, _u32p, C.c_uint32, C.c_int, C.c_uint64, _f32p, _f64p)
    f("orc_synth_edges", None, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_int,
      _u64p, _u64p, _u64p, _u64p, _u64p, C.c_int)
    if hasattr(L, "orc_p2_proto_marker"):
        from . import pyoracle_p2
        pyoracle_p2.proto(L, f)


# ------------------------------------------------------------------ small OO helpers ----------
class Hll:
    """HyperLogLog<N, FastHasher> (crates/core/src/hyperloglog.rs:4331-4547)."""

    def __init__(self, n=64):
        self.n = n
        self.registers = np.zeros(n, np.uint8)

    def add(self, item):
        lib().orc_hll_add(self.registers, self.n, int(item) & 0xFFFFFFFFFFFFFFFF)

    def merge(self, other):
        lib().orc_hll_merge(self.registers, other.registers, self.n)

    def size(self):
        return int(lib().orc_hll_size(self.registers, self.n))


def hll_size(regs):
    regs = np.ascontiguousarray(regs, np.uint8)
    return int(lib().orc_hll_size(regs, regs.size))


class KahanSum:
    def __init__(self):
        self._s = C.c_double(0.0)
        self._e = C.c_double(0.0)

    def add(self, x):
        lib().orc_kahan_add(C.byref(self._s), C.byref(self._e), float(x))

    @property
    def sum(self):
        return self._s.value

    @property
    def err(self):
        return self._e.value


class Bloom:
    def __init__(self, items, fp):
        self.h = lib().orc_bloom_new(items, fp)

    def insert(self, x):
        lib().orc_bloom_insert(self.h, x)

    def contains(self, x):
        return bool(lib().orc_bloom_contains(self.h, x))

    def estimate_card(self):
        return int(lib().orc_bloom_estimate_card(self.h))

    def __del__(self):
        try:
            lib().orc_bloom_free(self.h)
        except Exception:
            pass


def _edges(from_lo, from_hi, to_lo, to_hi, rel):
    arrs = [np.ascontiguousarray(a, np.uint64) for a in (from_lo, from_hi, to_lo, to_hi, rel)]
    n = arrs[0].size
    assert all(a.size == n for a in arrs)
    return arrs, n


def hyperball_faithful(from_lo, from_hi, to_lo, to_hi, rel, skip_mask=SKIPPED_REL_MASK, max_iters=0):
    """The reference-shaped single-threaded HyperBall.  Returns dict(ids_lo, ids_hi, centrality,
    n_nodes, iters) with ids ascending (u128) and only centrality > 0, like the BTreeMap of
    harmonic.rs:289-311."""
    arrs, n = _edges(from_lo, from_hi, to_lo, to_hi, rel)
    L = lib()
    h = L.orc_hb_faithful_run(*arrs, n, skip_mask, max_iters)
    try:
        k = L.orc_hb_faithful_len(h)
        lo = np.zeros(k, np.uint64); hi = np.zeros(k, np.uint64); c = np.zeros(k, np.float64)
        L.orc_hb_faithful_result(h, lo, hi, c)
        return dict(ids_lo=lo, ids_hi=hi, centrality=c, n_nodes=int(L.orc_hb_faithful_num_nodes(h)),
                    iters=int(L.orc_hb_faithful_iters(h)))
    finally:
        L.orc_hb_faithful_free(h)


class DenseHyperBall:
    """Flat-array HyperBall over dense ranks; steppable (parity checker for registers)."""

    def __init__(self, from_lo, from_hi, to_lo, to_hi, rel, skip_mask=SKIPPED_REL_MASK, threads=1, mt=False):
        """mt=True stages with all `threads` (oracle_hyperball_mt.cpp; same object, for 10^9-edge inputs)."""
        arrs, n = _edges(from_lo, from_hi, to_lo, to_hi, rel)
        self.L = lib()
        create = self.L.orc_hb_dense_create_mt if mt else self.L.orc_hb_dense_create
        self.h = create(*arrs, n, skip_mask, threads)
        if not self.h:
            raise ValueError("more than 2^32-1 nodes")
        self.n_nodes = int(self.L.orc_hb_dense_num_nodes(self.h))
        self.n_edges = int(self.L.orc_hb_dense_num_edges(self.h))

    def step(self):
        return int(self.L.orc_hb_dense_step(self.h))

    def reset(self):
        self.L.orc_hb_dense_reset(self.h)

    def num_self_loops(self):
        return int(self.L.orc_hb_dense_num_self_loops(self.h))

    def registers_view(self):
        """Zero-copy (n_nodes, 64) uint8 view of the current registers (valid until the next step / close)."""
        p = self.L.orc_hb_dense_registers_ptr(self.h)
        buf = (C.c_uint8 * (self.n_nodes * 64)).from_address(p)
        return np.frombuffer(buf, np.uint8).reshape(self.n_nodes, 64)

    def run(self, max_iters=0):
        return int(self.L.orc_hb_dense_run(self.h, max_iters))

    @property
    def iters(self):
        return int(self.L.orc_hb_dense_iters(self.h))

    def registers(self, first=0, count=None):
        count = self.n_nodes - first if count is None else count
        out = np.zeros((count, 64), np.uint8)
        if count:
            self.L.orc_hb_dense_registers(self.h, first, count, out)
        return out

    def ids(self):
        lo = np.zeros(self.n_nodes, np.uint64); hi = np.zeros(self.n_nodes, np.uint64)
        self.L.orc_hb_dense_ids(self.h, lo, hi)
        return lo, hi

    def kahan(self):
        s = np.zeros(self.n_nodes, np.float64); e = np.zeros(self.n_nodes, np.float64)
        self.L.orc_hb_dense_kahan(self.h, s, e)
        return s, e

    def result(self):
        k = int(self.L.orc_hb_dense_result(self.h, None, None, None))
        lo = np.zeros(k, np.uint64); hi = np.zeros(k, np.uint64); c = np.zeros(k, np.float64)
        if k:
            self.L.orc_hb_dense_result(self.h, lo.ctypes.data, hi.ctypes.data, c.ctypes.data)
        return dict(ids_lo=lo, ids_hi=hi, centrality=c, n_nodes=self.n_nodes, iters=self.iters)

    def close(self):
        if self.h:
            self.L.orc_hb_dense_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def synth_edges(kind, n_nodes, n_edges, seed=42, scale=26, first=0, threads=1):
    """CPU port of the repo's synthetic edge generator (stract_b200/synth.py, csrc/synth.cu): kind 0 = uniform
    (configs[0]), 1 = R-MAT (configs[1]).  Returns dict(from_lo, from_hi, to_lo, to_hi, rel_flags)."""
    a = [np.empty(n_edges, np.uint64) for _ in range(5)]
    lib().orc_synth_edges(kind, n_nodes, first, n_edges, seed, scale, *a, threads)
    return dict(from_lo=a[0], from_hi=a[1], to_lo=a[2], to_hi=a[3], rel_flags=a[4])


def graph_links(from_lo, from_hi, to_lo, to_hi, rel, skip_mask=0):
    """(ids_lo, ids_hi, from_rank, to_rank): the unique links that pass `skip_mask` (first occurrence decides, like the
    Webgraph iterator) over dense node ranks -- the input of graph_distances / approx_harmonic.  numpy, test sizes only."""
    flo = np.asarray(from_lo, np.uint64); fhi = np.asarray(from_hi, np.uint64); tlo = np.asarray(to_lo, np.uint64); thi = np.asarray(to_hi, np.uint64)
    ids = np.unique(np.concatenate([np.stack([fhi, flo], 1), np.stack([thi, tlo], 1)]), axis=0)
    order = {(int(h), int(l)): i for i, (h, l) in enumerate(ids)}
    fr = np.array([order[(int(h), int(l))] for h, l in zip(fhi, flo)], np.uint32)
    tr = np.array([order[(int(h), int(l))] for h, l in zip(thi, tlo)], np.uint32)
    pair = fr.astype(np.uint64) << np.uint64(32) | tr.astype(np.uint64)
    _, first = np.unique(pair, return_index=True)
    first.sort()
    keep = (np.asarray(rel, np.uint64)[first] & np.uint64(skip_mask)) == 0
    first = first[keep]
    return ids[:, 1].copy(), ids[:, 0].copy(), fr[first], tr[first]


def graph_distances(n, from_rank, to_rank, sources, groups=None, max_dist=None, reversed=False):
    """dijkstra_multi (webgraph/shortest_path.rs:57-105) per group of sources: uint8 [n_groups, n], 255 = not reached."""
    fr = np.ascontiguousarray(from_rank, np.uint32); tr = np.ascontiguousarray(to_rank, np.uint32)
    src = np.ascontiguousarray(sources, np.uint32)
    grp = np.arange(src.size, dtype=np.uint32) if groups is None else np.ascontiguousarray(groups, np.uint32)
    ng = int(grp.max()) + 1 if grp.size else 1
    out = np.zeros((ng, n), np.uint8)
    lib().orc_graph_distances(n, fr, tr, fr.size, src, grp, src.size, ng, -1 if max_dist is None else int(max_dist), 1 if reversed else 0, out.reshape(-1))
    return out


def approx_harmonic(n, from_rank, to_rank, sources, max_dist=7, num_nodes=None):
    """ApproxHarmonic::build for a fixed sample: (f32 sums in source order, f64 sums of the same f32 terms), 0 = not reached.
    A source rank 0xFFFFFFFF (an id that is not a node) counts in the sample size and reaches nothing."""
    fr = np.ascontiguousarray(from_rank, np.uint32); tr = np.ascontiguousarray(to_rank, np.uint32)
    src = np.ascontiguousarray(sources, np.uint32)
    o32 = np.zeros(n, np.float32); o64 = np.zeros(n, np.float64)
    lib().orc_approx_harmonic(n, fr, tr, fr.size, src, src.size, int(max_dist), int(n if num_nodes is None else num_nodes), o32, o64)
    return o32, o64


def inbound_similarity(ids_lo, ids_hi, from_rank, to_rank, liked, disliked, candidates, normalized=False, self_score=1.0):
    """inbound_similarity::Scorer::score for every candidate (ranks; 0xFFFFFFFF = not a node of the graph)."""
    lo = np.ascontiguousarray(ids_lo, np.uint64); hi = np.ascontiguousarray(ids_hi, np.uint64)
    fr = np.ascontiguousarray(from_rank, np.uint32); tr = np.ascontiguousarray(to_rank, np.uint32)
    li = np.ascontiguousarray(liked, np.uint32); di = np.ascontiguousarray(disliked, np.uint32); ca = np.ascontiguousarray(candidates, np.uint32)
    out = np.zeros(ca.size, np.float64)
    lib().orc_inbound_similarity(lo.size, lo, hi, fr, tr, fr.size, li, li.size, di, di.size, ca, ca.size, 1 if normalized else 0, float(self_score), out)
    return out


def harmonic_ranks(ids_lo, ids_hi, values, ties_desc=False):
    """Order of store_harmonic's rank pass (crates/core/src/webgraph/centrality/mod.rs:88-108): sort by
    (Reverse(SortableFloat(centrality)), node_id) -- centrality descending under total_cmp, node id ascending; with
    ties_desc the order of top_nodes (mod.rs:17-37): the largest (centrality, node_id) pairs first.  Returns the
    permutation of the input (test infrastructure, numpy)."""
    import numpy as np
    lo = np.asarray(ids_lo, np.uint64); hi = np.asarray(ids_hi, np.uint64); v = np.asarray(values, np.float64)
    bits = v.view(np.uint64)
    key = np.where(bits >> np.uint64(63), ~bits, bits | np.uint64(1 << 63))   # total_cmp order as unsigned integers
    if ties_desc:
        return np.lexsort((~lo, ~hi, ~key))
    return np.lexsort((lo, hi, ~key))
