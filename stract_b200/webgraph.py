"""Host-side mirror of the reference's webgraph-centrality interface, backed by libstract_b200.so.

Mirrors (same names / argument meaning / behaviour):
  RelFlags, SKIPPED_REL           crates/core/src/webpage/html/links.rs:114-141, harmonic.rs:36-49
  Edge / Webgraph.insert/commit/host_edges/host_nodes
                                  crates/core/src/webgraph/{edge.rs:30-35,mod.rs:157-194}
  HarmonicCentrality.calculate/get/iter/len
                                  crates/core/src/webgraph/centrality/harmonic.rs:289-311
  Betweenness.calculate           crates/core/src/webgraph/centrality/betweenness.rs:29-175
  ShardedHarmonicCentrality       the AMPC job (entrypoint/ampc/harmonic_centrality/*): one process
                                  per GPU, the DHT max-upsert replaced by an all-gather of owned rows

NodeID is a python int holding the u128 (crates/core/src/webgraph/node.rs:37).  All compute runs in
the CUDA library; this module only marshals buffers.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import GraphInfo, IterStats, check, lib
from ._hostmem import host_out


class RelFlags:
    ALTERNATE = 1 << 0; AUTHOR = 1 << 1; CANONICAL = 1 << 2; HELP = 1 << 3; ICON = 1 << 4
    LICENSE = 1 << 5; ME = 1 << 6; NEXT = 1 << 7; NOFOLLOW = 1 << 8; PREV = 1 << 9
    PRIVACY_POLICY = 1 << 10; SEARCH = 1 << 11; STYLESHEET = 1 << 12; TAG = 1 << 13
    TERMS_OF_SERVICE = 1 << 14; SPONSORED = 1 << 15; IS_IN_FOOTER = 1 << 16
    IS_IN_NAVIGATION = 1 << 17; LINK_TAG = 1 << 18; SCRIPT_TAG = 1 << 19; META_TAG = 1 << 20
    SAME_ICANN_DOMAIN = 1 << 21; UGC = 1 << 22


SKIPPED_REL = (RelFlags.TAG | RelFlags.NOFOLLOW | RelFlags.SPONSORED | RelFlags.IS_IN_FOOTER
               | RelFlags.IS_IN_NAVIGATION | RelFlags.PRIVACY_POLICY | RelFlags.TERMS_OF_SERVICE
               | RelFlags.SEARCH | RelFlags.LINK_TAG | RelFlags.SCRIPT_TAG | RelFlags.SAME_ICANN_DOMAIN
               | RelFlags.UGC)
assert SKIPPED_REL == 0x6FED00

_M64 = (1 << 64) - 1


class Edge:
    """SmallEdge{from, to, rel_flags} (crates/core/src/webgraph/edge.rs:30-35)."""
    __slots__ = ("from_", "to", "rel_flags")

    def __init__(self, from_, to, rel_flags=0):
        self.from_, self.to, self.rel_flags = int(from_), int(to), int(rel_flags)

    @classmethod
    def new_test(cls, from_, to):  # Edge::new_test, edge.rs:198-206
        return cls(from_, to, 0)


def _ptr(a):
    """(pointer, keepalive) of a numpy array or a torch tensor (host or cuda), dtype uint64/int64."""
    if a is None:
        return None, None
    if hasattr(a, "data_ptr"):  # torch tensor
        assert a.is_contiguous() and a.element_size() == 8
        return a.data_ptr(), a
    a = np.ascontiguousarray(a, np.uint64)
    return a.ctypes.data, a


class Webgraph:
    """A host graph as the stream `Webgraph::host_edges()` yields it (SoA of from/to/rel_flags).

    Built either edge by edge (`insert` + `commit`, like the reference's tests) or from arrays
    (`from_arrays`; numpy or torch tensors, host or already resident in HBM)."""

    def __init__(self):
        self._pending = []
        self.from_lo = self.from_hi = self.to_lo = self.to_hi = self.rel = None
        self.n_edges = 0

    @classmethod
    def from_arrays(cls, from_lo, from_hi, to_lo, to_hi, rel_flags):
        g = cls()
        g.from_lo, g.from_hi, g.to_lo, g.to_hi, g.rel = from_lo, from_hi, to_lo, to_hi, rel_flags
        g.n_edges = int(from_lo.shape[0]) if hasattr(from_lo, "shape") else len(from_lo)
        return g

    def insert(self, edge):
        self._pending.append(edge)

    def commit(self):
        if not self._pending:
            return
        n = len(self._pending)
        cols = [np.zeros(n, np.uint64) for _ in range(5)]
        for i, e in enumerate(self._pending):
            cols[0][i] = e.from_ & _M64; cols[1][i] = e.from_ >> 64
            cols[2][i] = e.to & _M64; cols[3][i] = e.to >> 64
            cols[4][i] = e.rel_flags
        if self.n_edges:
            old = [np.asarray(a, np.uint64) for a in (self.from_lo, self.from_hi, self.to_lo, self.to_hi, self.rel)]
            cols = [np.concatenate([o, c]) for o, c in zip(old, cols)]
        self.from_lo, self.from_hi, self.to_lo, self.to_hi, self.rel = cols
        self.n_edges = len(cols[0])
        self._pending = []

    def host_edges(self):
        """Iterate SmallEdge (host arrays only; debugging aid -- the library consumes the arrays)."""
        for i in range(self.n_edges):
            yield Edge((int(self.from_hi[i]) << 64) | int(self.from_lo[i]),
                       (int(self.to_hi[i]) << 64) | int(self.to_lo[i]), int(self.rel[i]))

    def host_nodes(self):
        s = set()
        for e in self.host_edges():
            s.add(e.from_); s.add(e.to)
        return s


class DeviceGraph:
    """Owner of an `sb200_graph*`: the staged CSR + HyperBall state in HBM."""

    def __init__(self, graph, device=0, rank=0, world_size=1, skipped_rel=SKIPPED_REL):
        self._h = C.c_void_p()
        self._L = lib()
        graph.commit()
        ptrs = [_ptr(a) for a in (graph.from_lo, graph.from_hi, graph.to_lo, graph.to_hi, graph.rel)]
        self._keep = [p[1] for p in ptrs]
        check(self._L.sb200_graph_create(*(p[0] for p in ptrs), graph.n_edges, skipped_rel, device, rank,
                                         world_size, C.byref(self._h)))
        self._keep = None
        self.world_size, self.rank, self.device = world_size, rank, device
        self.p2p = False

    def info(self):
        gi = GraphInfo()
        check(self._L.sb200_graph_get_info(self._h, C.byref(gi)))
        return {k: getattr(gi, k) for k, _ in GraphInfo._fields_}

    def reset(self):
        check(self._L.sb200_hyperball_reset(self._h))

    def set_option(self, name, value):
        """Tuning switch of this handle: "quad_side_ctas", "owned_items", "publish_all", "l2_window_mb" (the persisting L2
        window over the head of the register array, in MiB; 0 turns it off), "l1_hub_kb" (the pulls' L1 budget for hub
        sources, in KiB; 0 sends every gather around L1) (sb200_hyperball_set_option)."""
        check(self._L.sb200_hyperball_set_option(self._h, name.encode(), float(value)))

    def set_policy(self, dense_frac=-1.0, push_div=-1.0, force_mode=-1):
        check(self._L.sb200_hyperball_set_policy(self._h, dense_frac, push_div, force_mode))

    def step(self):
        st = IterStats()
        check(self._L.sb200_hyperball_step(self._h, C.byref(st)))
        return {k: getattr(st, k) for k, _ in IterStats._fields_}

    def run(self, max_iters=0, cap=256):
        done = C.c_uint32(0)
        arr = (IterStats * cap)()
        check(self._L.sb200_hyperball_run(self._h, max_iters, C.byref(done), arr, cap))
        n = min(done.value, cap)
        return done.value, [{k: getattr(arr[i], k) for k, _ in IterStats._fields_} for i in range(n)]

    def last_run_ms(self):
        ms = C.c_float(0)
        check(self._L.sb200_hyperball_last_run_ms(self._h, C.byref(ms)))
        return ms.value

    def set_profiling(self, on=True):
        check(self._L.sb200_hyperball_set_profiling(self._h, 1 if on else 0))

    def profile(self):
        arr = (_lib.KernelProf * 16)()
        n = C.c_uint32(0)
        check(self._L.sb200_hyperball_get_profile(self._h, arr, 16, C.byref(n)))
        return [dict(name=arr[i].name.decode(), launches=arr[i].launches, ms=arr[i].ms, alg_bytes=arr[i].alg_bytes)
                for i in range(n.value)]

    def result(self):
        # one call with capacity = node count (an upper bound on the nodes with centrality > 0) instead of a
        # count-only call followed by a second pass; big outputs land in page-locked memory (_hostmem.py)
        import time
        n = self.info()["n_nodes"]
        ln = C.c_uint64(0)
        t0 = time.perf_counter()
        lo = host_out(n, np.uint64); hi = host_out(n, np.uint64); c = host_out(n, np.float64)
        t1 = time.perf_counter()
        if n:
            check(self._L.sb200_hyperball_result(self._h, lo.ctypes.data, hi.ctypes.data, c.ctypes.data, n, C.byref(ln)))
        self.result_wall_ms = {"host_alloc": (t1 - t0) * 1e3, "call": (time.perf_counter() - t1) * 1e3}
        k = ln.value
        return lo[:k], hi[:k], c[:k]

    def ranked(self, ties_desc=False, limit=None):
        """Nodes with centrality > 0 in rank order: centrality descending (f64 total order), ties by node id ascending
        (entry i has harmonic rank i, store_harmonic, webgraph/centrality/mod.rs:88-108) or -- ties_desc -- descending
        (top_nodes' order, mod.rs:17-37).  `limit` keeps the leading entries only."""
        n = self.info()["n_nodes"]
        cap = n if limit is None else min(int(limit), n)
        ln = C.c_uint64(0)
        lo = host_out(cap, np.uint64); hi = host_out(cap, np.uint64); c = host_out(cap, np.float64)
        check(self._L.sb200_hyperball_ranked(self._h, 1 if ties_desc else 0, lo.ctypes.data if cap else None,
                                              hi.ctypes.data if cap else None, c.ctypes.data if cap else None, cap, C.byref(ln)))
        k = min(ln.value, cap)
        return lo[:k], hi[:k], c[:k], ln.value

    def registers(self, first=0, count=None):
        n = self.info()["n_nodes"]
        count = n - first if count is None else count
        out = np.zeros((count, 64), np.uint8)
        if count:
            check(self._L.sb200_hyperball_registers(self._h, first, count, out.ctypes.data))
        return out

    def kahan(self, first=0, count=None):
        n = self.info()["n_nodes"]
        count = n - first if count is None else count
        s = np.zeros(count, np.float64); e = np.zeros(count, np.float64)
        if count:
            check(self._L.sb200_hyperball_kahan(self._h, first, count, s.ctypes.data, e.ctypes.data))
        return s, e

    def node_ids(self):
        n = self.info()["n_nodes"]
        lo = np.zeros(n, np.uint64); hi = np.zeros(n, np.uint64)
        if n:
            check(self._L.sb200_graph_node_ids(self._h, 0, n, lo.ctypes.data, hi.ctypes.data))
        return lo, hi

    def row_ranges(self):
        b = (C.c_uint64 * (self.world_size + 1))()
        check(self._L.sb200_graph_row_ranges(self._h, b))
        return list(b)

    def exchange_ptrs(self):
        regs, fr = C.c_void_p(), C.c_void_p()
        rb, fb = C.c_uint64(), C.c_uint64()
        check(self._L.sb200_hyperball_exchange_ptrs(self._h, C.byref(regs), C.byref(rb), C.byref(fr), C.byref(fb)))
        return regs.value, rb.value, fr.value, fb.value

    def exchange_tensors(self):
        """(registers uint8 [N*64], changed bitmap int32 [ceil(N/32)]) as zero-copy torch views of HBM."""
        import torch
        regs, rb, fr, fb = self.exchange_ptrs()
        dev = torch.device("cuda", self.device)
        torch.cuda.synchronize(dev)
        return _as_tensor(regs, rb, torch.uint8, dev), _as_tensor(fr, fb, torch.int32, dev)

    def enable_p2p(self, group=None):
        """Fused exchange: swap CUDA IPC handles with every other rank and let the pull kernels store produced rows
        straight into the peers' replicas over NVLink (sb200_hyperball_ipc_*)."""
        import torch.distributed as dist
        mine = (C.c_uint8 * _lib.IPC_BLOB_BYTES)()
        check(self._L.sb200_hyperball_ipc_export(self._h, mine))
        allh = [None] * self.world_size
        dist.all_gather_object(allh, bytes(mine), group=group)
        for r, h in enumerate(allh):
            if r == self.rank:
                continue
            buf = (C.c_uint8 * _lib.IPC_BLOB_BYTES).from_buffer_copy(h)
            check(self._L.sb200_hyperball_ipc_import(self._h, buf))
        check(self._L.sb200_hyperball_p2p_enable(self._h, 1))
        dist.barrier(group=group)
        self.p2p = True

    def enable_symmetric(self, group=None, multicast=True):
        """Fused exchange over torch symmetric memory: the register arrays and bitmaps move into buffers that every
        rank maps (and, on an NVSwitch box, that are bound to a multicast object).  With `multicast` and switch
        support a produced row is stored once, to the multicast address, and the switch replicates it into every
        replica; otherwise it is stored to each peer mapping like `enable_p2p` does.  Returns "multicast" or
        "unicast".  The buffers are torch tensors owned by this object (plumbing; the stores are the library's)."""
        import torch
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        grp = group if group is not None else dist.group.WORLD
        rb, bb = C.c_uint64(0), C.c_uint64(0)
        check(self._L.sb200_hyperball_state_bytes(self._h, C.byref(rb), C.byref(bb)))
        dev = torch.device("cuda", self.device)
        bufs = [symm.empty(rb.value, dtype=torch.uint8, device=dev), symm.empty(rb.value, dtype=torch.uint8, device=dev),
                symm.empty(bb.value // 4, dtype=torch.int32, device=dev), symm.empty(bb.value // 4, dtype=torch.int32, device=dev)]
        hdls = [symm.rendezvous(b, grp) for b in bufs]
        torch.cuda.synchronize(dev)
        check(self._L.sb200_hyperball_bind_state(self._h, *(b.data_ptr() for b in bufs)))
        use_mc = bool(multicast) and all(int(getattr(h, "multicast_ptr", 0) or 0) != 0 for h in hdls)
        if use_mc:
            cols = [[int(h.multicast_ptr)] for h in hdls]
        else:
            cols = [[int(p) for r, p in enumerate(h.buffer_ptrs) if r != hdls[0].rank] for h in hdls]
        n = len(cols[0])
        arrs = [(C.c_uint64 * max(n, 1))(*c) for c in cols]
        check(self._L.sb200_hyperball_set_publish_targets(self._h, n, *arrs))
        self._symm = (bufs, hdls)  # keep the buffers alive for as long as the handle uses them
        dist.barrier(group=group)
        self.p2p = True
        return "multicast" if use_mc else "unicast"

    def run_sharded(self, max_iters=0, cap=256):
        """The whole round loop behind the ABI (sb200_hyperball_run_sharded): all ranks call it together after
        enable_p2p(); the ranks meet in a device-side barrier that also sums the changed counts (no NCCL)."""
        done = C.c_uint32(0)
        arr = (IterStats * cap)()
        check(self._L.sb200_hyperball_run_sharded(self._h, max_iters, C.byref(done), arr, cap))
        n = min(done.value, cap)
        return done.value, [{k: getattr(arr[i], k) for k, _ in IterStats._fields_} for i in range(n)]

    def ownership(self):
        """(owned uint8[N], subscribers uint32[N]) in ascending-id order (sb200_graph_ownership)."""
        n = self.info()["n_nodes"]
        o = np.zeros(n, np.uint8); m = np.zeros(n, np.uint32)
        if n:
            check(self._L.sb200_graph_ownership(self._h, o.ctypes.data, m.ctypes.data))
        return o, m

    def distances(self, sources, groups=None, max_dist=0, reversed=False):
        """dijkstra_multi with unit costs (webgraph/shortest_path.rs:57-105): `sources` = node ids (python ints), `groups[i]` =
        the search source i belongs to (default: one search per source).  Returns uint8 [n_groups, n_nodes] in ascending-id
        order, 255 = not reached; with max_dist > 0 distances up to max_dist + 1 are reported like the reference does."""
        n = self.info()["n_nodes"]
        lo = np.array([int(x) & _M64 for x in sources], np.uint64); hi = np.array([int(x) >> 64 for x in sources], np.uint64)
        grp = np.arange(len(lo), dtype=np.uint32) if groups is None else np.ascontiguousarray(groups, np.uint32)
        ng = int(grp.max()) + 1 if len(grp) else 1
        out = np.full((ng, n), 255, np.uint8)
        check(self._L.sb200_graph_distances(self._h, lo.ctypes.data, hi.ctypes.data, grp.ctypes.data, len(lo), ng, int(max_dist),
                                            1 if reversed else 0, out.ctypes.data))
        return out

    def approx_harmonic(self, sources, max_dist=7, num_nodes=0):
        """ApproxHarmonic::build for the given sample (webgraph/centrality/approx_harmonic.rs:40-88): (ids_lo, ids_hi, centrality)
        of the reached nodes in ascending id order."""
        n = self.info()["n_nodes"]
        lo = np.array([int(x) & _M64 for x in sources], np.uint64); hi = np.array([int(x) >> 64 for x in sources], np.uint64)
        ln = C.c_uint64(0)
        olo = host_out(n, np.uint64); ohi = host_out(n, np.uint64); oc = host_out(n, np.float64)
        check(self._L.sb200_approx_harmonic(self._h, lo.ctypes.data, hi.ctypes.data, len(lo), int(max_dist), int(num_nodes),
                                            olo.ctypes.data if n else None, ohi.ctypes.data if n else None, oc.ctypes.data if n else None, n, C.byref(ln)))
        k = ln.value
        return olo[:k], ohi[:k], oc[:k]

    def betweenness(self, sources):
        """Betweenness::calculate for the given sources, in the given order (webgraph/centrality/betweenness.rs:29-146):
        (ids_lo, ids_hi, centrality, max_dist) over the sources and the nodes they reach, in ascending id order.  Create the
        handle with skipped_rel=0: the reference's ForwardlinksQuery sees every link."""
        n = self.info()["n_nodes"]
        lo = np.array([int(x) & _M64 for x in sources], np.uint64); hi = np.array([int(x) >> 64 for x in sources], np.uint64)
        ln = C.c_uint64(0); md = C.c_uint32(0)
        olo = host_out(n, np.uint64); ohi = host_out(n, np.uint64); oc = host_out(n, np.float64)
        check(self._L.sb200_betweenness(self._h, lo.ctypes.data, hi.ctypes.data, len(lo), olo.ctypes.data if n else None,
                                        ohi.ctypes.data if n else None, oc.ctypes.data if n else None, n, C.byref(ln), C.byref(md)))
        k = ln.value
        return olo[:k], ohi[:k], oc[:k], md.value

    def inbound_similarity(self, liked, disliked, candidates, normalized=False, self_score=1.0):
        """inbound_similarity::Scorer over the resident graph (ranking/inbound_similarity.rs:71-119): one f64 score per candidate."""
        def split(ids):
            return (np.array([int(x) & _M64 for x in ids], np.uint64), np.array([int(x) >> 64 for x in ids], np.uint64))
        ll, lh = split(liked); dl, dh = split(disliked); cl, ch = split(candidates)
        out = np.zeros(len(cl), np.float64)
        check(self._L.sb200_inbound_similarity(self._h, ll.ctypes.data, lh.ctypes.data, len(ll), dl.ctypes.data, dh.ctypes.data, len(dl),
                                               cl.ctypes.data, ch.ctypes.data, len(cl), 1 if normalized else 0, float(self_score), out.ctypes.data))
        return out

    def exchange_done(self, global_n_changed):
        check(self._L.sb200_hyperball_exchange_done(self._h, int(global_n_changed)))

    def close(self):
        if self._h:
            self._L.sb200_graph_destroy(self._h)
            self._h = C.c_void_p()
        self._symm = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DeviceGroup:
    """n ranks of the sharded path driven by ONE process (sb200_hyperball_group_link / _group_run): the n GPUs of a
    box, or -- `devices` repeating an index -- several ranks on one GPU (how the 1-GPU test box exercises the fused
    exchange).  Replaces the AMPC coordinator + workers + DHT of entrypoint/ampc/harmonic_centrality/."""

    def __init__(self, graph, devices, skipped_rel=SKIPPED_REL):
        self.world = len(devices)
        self.ranks = [DeviceGraph(graph, device=d, rank=r, world_size=self.world, skipped_rel=skipped_rel) for r, d in enumerate(devices)]
        self._L = lib()
        self._arr = (C.c_void_p * self.world)(*[h._h for h in self.ranks])
        check(self._L.sb200_hyperball_group_link(self._arr, self.world))

    def reset(self):
        for h in self.ranks:
            h.reset()

    def run(self, max_iters=0, cap=256):
        done = C.c_uint32(0)
        arr = (IterStats * (cap * self.world))()
        check(self._L.sb200_hyperball_group_run(self._arr, self.world, max_iters, C.byref(done), arr, cap))
        n = min(done.value, cap)
        return done.value, [[{k: getattr(arr[r * cap + i], k) for k, _ in IterStats._fields_} for i in range(n)] for r in range(self.world)]

    def result(self):
        """The union of the ranks' owned results in ascending id order (what HarmonicCentrality.iter() yields)."""
        parts = [h.result() for h in self.ranks]
        lo = np.concatenate([p[0] for p in parts]); hi = np.concatenate([p[1] for p in parts]); c = np.concatenate([p[2] for p in parts])
        order = np.lexsort((lo, hi))
        return lo[order], hi[order], c[order]

    def close(self):
        for h in self.ranks:
            h.close()


class HarmonicCentrality:
    """`HarmonicCentrality(BTreeMap<NodeID, f64>)` (harmonic.rs:289-311): ascending node id, nodes with
    zero centrality absent."""

    def __init__(self, ids_lo, ids_hi, values, n_nodes=0, iterations=0, stats=None, info=None):
        self.ids_lo, self.ids_hi, self.values = ids_lo, ids_hi, values
        self.n_nodes, self.iterations, self.stats, self.info = n_nodes, iterations, stats or [], info or {}
        self._map = None

    @classmethod
    def calculate(cls, graph, device=0, max_iters=0, with_ranks=False, top=1_000_000):
        import time
        t0 = time.perf_counter()
        dg = DeviceGraph(graph, device=device)
        try:
            t1 = time.perf_counter()
            iters, stats = dg.run(max_iters)
            t2 = time.perf_counter()
            lo, hi, c = dg.result()
            t3 = time.perf_counter()
            info = dg.info()
            ranks = None
            if with_ranks:   # Centrality::build_harmonic: store_harmonic's rank pass + top_nodes (entrypoint/centrality.rs:41-71)
                rlo, rhi, _, _ = dg.ranked(False)
                tlo, thi, tc, _ = dg.ranked(True, limit=top)
                ranks = ((rlo, rhi), (tlo, thi, tc))
        finally:
            dg.close()
        t4 = time.perf_counter()
        # host wall clock of the four C-ABI phases (every call returns synchronised)
        info["wall_ms"] = {"create": (t1 - t0) * 1e3, "run": (t2 - t1) * 1e3, "result": (t3 - t2) * 1e3,
                           "destroy": (t4 - t3) * 1e3, **{"result_" + k: v for k, v in dg.result_wall_ms.items()}}
        r = cls(lo, hi, c, info["n_nodes"], iters, stats, info)
        if ranks:
            r.rank_ids, r.top = ranks
        return r

    def harmonic_rank(self):
        """{node id: rank} as store_harmonic writes it into the `harmonic_rank` store (needs calculate(..., with_ranks=True))."""
        lo, hi = self.rank_ids
        return {(int(h) << 64) | int(l): i for i, (l, h) in enumerate(zip(lo, hi))}

    def top_nodes(self, k):
        """top_nodes(store, TopNodes::Top(k)): [(node id, centrality)], (centrality, id) descending."""
        lo, hi, c = self.top
        return [((int(h) << 64) | int(l), float(v)) for l, h, v in zip(lo[:k], hi[:k], c[:k])]

    def _m(self):
        if self._map is None:
            self._map = {(int(h) << 64) | int(l): float(v) for l, h, v in zip(self.ids_lo, self.ids_hi, self.values)}
        return self._map

    def get(self, node):
        return self._m().get(int(node))

    def iter(self):
        for l, h, v in zip(self.ids_lo, self.ids_hi, self.values):
            yield (int(h) << 64) | int(l), float(v)

    def __len__(self):
        return len(self.values)

    def len(self):
        return len(self.values)

    def is_empty(self):
        return len(self.values) == 0


class Betweenness:
    """`Betweenness { centrality: HashMap<Node, f64>, max_dist }` (webgraph/centrality/betweenness.rs:149-175).

    The reference takes the first 100 000 nodes of an FxHashSet as sources; here `sources=None` means every node when the
    graph has at most MAX_SOURCES of them (the reference's source set), otherwise the first MAX_SOURCES in ascending id."""
    MAX_SOURCES = 100_000

    def __init__(self, ids_lo, ids_hi, values, max_dist):
        self.ids_lo, self.ids_hi, self.values, self.max_dist = ids_lo, ids_hi, values, max_dist
        self.centrality = {(int(h) << 64) | int(l): float(v) for l, h, v in zip(ids_lo, ids_hi, values)}

    @classmethod
    def calculate(cls, graph, device=0, sources=None):
        dg = DeviceGraph(graph, device=device, skipped_rel=0)   # ForwardlinksQuery applies no rel-flag filter
        try:
            if sources is None:
                lo, hi = dg.node_ids()
                sources = [(int(h) << 64) | int(l) for l, h in zip(lo[:cls.MAX_SOURCES], hi[:cls.MAX_SOURCES])]
            return cls(*dg.betweenness(sources))
        finally:
            dg.close()


def run_sharded_loop(engine, world_size, group=None, max_iters=0):
    """The AMPC round loop (crates/core/src/ampc/coordinator.rs:151-213 driving the six CentralityMappers,
    entrypoint/ampc/harmonic_centrality/mapper.rs:38-45) for one rank, with torch.distributed as transport.

    `engine` owns this rank's shard: `step()` runs one HyperBall iteration over its destination rows,
    `exchange_tensors()` exposes the full register array and changed bitmap as torch tensors.  After each step
    every owner broadcasts its rows (the DHT `HyperLogLog64Upsert` max-merge has a single writer per row, so it is
    an all-gather) and its bitmap words (SaveBloom/UpdateBloom), and the changed counts are summed
    (Meta.round_had_changes)."""
    import torch
    import torch.distributed as dist
    stats = []
    t = 0
    fused = bool(getattr(engine, "p2p", False))
    if fused:
        dist.barrier(group=group)  # every replica must be (re)initialised before a peer may write into it
    while True:
        st = engine.step()
        if fused:
            # rows and changed bits already sit in every replica; the all-reduce is the inter-step barrier
            dev = torch.device("cuda", engine.device)
            cnt = torch.tensor([st["n_changed"]], dtype=torch.int64, device=dev)
            dist.all_reduce(cnt, group=group)
            total = int(cnt.item())
            engine.exchange_done(total)
            st["n_changed_global"] = total
            stats.append(st)
            t += 1
            if total == 0 or (max_iters and t >= max_iters):
                return t, stats
            continue
        regs, fr = engine.exchange_tensors()
        cnt = torch.tensor([st["n_changed"]], dtype=torch.int64, device=regs.device)
        # Rows are owned in interleaved 32-row blocks, so the merge is the DHT's own operator: elementwise byte
        # max over all replicas (`HyperLogLog64Upsert`, ampc/dht/upsert.rs:66-83; registers only grow, a non-owner's
        # copy of a row is an older, smaller-or-equal state).  Each 32-bit bitmap word has a single owner too.
        fr8 = fr.view(torch.uint8)
        works = [dist.all_reduce(regs, op=dist.ReduceOp.MAX, group=group, async_op=True),
                 dist.all_reduce(fr8, op=dist.ReduceOp.MAX, group=group, async_op=True)]
        works.append(dist.all_reduce(cnt, group=group, async_op=True))
        for w in works:
            w.wait()
        if regs.is_cuda:
            torch.cuda.current_stream(regs.device).synchronize()
        total = int(cnt.item())
        engine.exchange_done(total)
        st["n_changed_global"] = total
        stats.append(st)
        t += 1
        if total == 0 or (max_iters and t >= max_iters):
            return t, stats


def shard_bounds(n_edges, rank, world_size):
    """The contiguous slice of an edge stream rank `rank` ingests (equal `ceil(E / world)` slices, the last ones shorter)."""
    chunk = -(-int(n_edges) // int(world_size)) if n_edges else 0
    return min(rank * chunk, n_edges), min((rank + 1) * chunk, n_edges)


def gather_edge_shards(shard, device, world_size, group=None):
    """Every rank holds ONE shard of the edge stream on its host -- as the reference's workers each hold one webgraph
    shard (entrypoint/ampc/harmonic_centrality/worker.rs) -- and needs the whole stream in HBM for the (replicated)
    staging.  Each rank copies its shard over ITS OWN PCIe link and an all-gather over NVLink/NVSwitch assembles the
    stream in rank order on every GPU: the stream crosses PCIe once in total instead of once per rank.

    `shard`: Webgraph over host arrays (numpy uint64 / torch int64, ideally page-locked).  `device`: CUDA index, or "cpu"
    (gloo; the host-logic tests).  Returns a Webgraph over device-resident arrays holding all shards concatenated."""
    import torch
    import torch.distributed as dist
    dev = torch.device("cpu") if device == "cpu" else torch.device("cuda", int(device))
    cuda = dev.type == "cuda"

    def as_i64(a):
        if isinstance(a, torch.Tensor):
            return a.view(torch.int64) if a.dtype != torch.int64 else a
        return torch.from_numpy(np.ascontiguousarray(a, np.uint64).view(np.int64))
    cols = [as_i64(a) if shard.n_edges else torch.zeros(0, dtype=torch.int64) for a in (shard.from_lo, shard.from_hi, shard.to_lo, shard.to_hi, shard.rel)]
    n_local = int(shard.n_edges)
    counts = torch.tensor([n_local], dtype=torch.int64, device=dev)
    all_counts = torch.zeros(world_size, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(all_counts, counts, group=group)
    all_counts = [int(x) for x in all_counts.tolist()]
    chunk = max(all_counts) if all_counts else 0
    total = sum(all_counts)
    if chunk == 0:
        z = torch.zeros(0, dtype=torch.int64, device=dev)
        return Webgraph.from_arrays(z, z, z, z, z)
    # the gathered layout is already the concatenation iff every shard but the trailing ones is full
    prefix_ok = all(all_counts[r] == chunk or sum(all_counts[r + 1:]) == 0 for r in range(world_size))
    copy_s = torch.cuda.Stream(device=dev) if cuda else None
    pending = []
    for c in cols:
        sl = torch.empty(chunk, dtype=torch.int64, device=dev)
        out = torch.empty(world_size * chunk, dtype=torch.int64, device=dev)
        if cuda:
            copy_s.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(copy_s):
                if n_local:
                    sl[:n_local].copy_(c, non_blocking=True)
                if n_local < chunk:
                    sl[n_local:].zero_()
            torch.cuda.current_stream(dev).wait_stream(copy_s)   # orders only the work queued so far: later copies overlap the gather
            sl.record_stream(copy_s)
        else:
            sl[:n_local] = c
            sl[n_local:] = 0
        pending.append((dist.all_gather_into_tensor(out, sl, group=group, async_op=True), out, sl))
    full = []
    for work, out, sl in pending:
        work.wait()
        if prefix_ok:
            full.append(out[:total])
        else:
            full.append(torch.cat([out[r * chunk: r * chunk + all_counts[r]] for r in range(world_size)]))
    del pending
    if cuda:
        torch.cuda.current_stream(dev).synchronize()   # the library stages on its own stream: the stream must be complete before it reads
    return Webgraph.from_arrays(*full)


class ShardedHarmonicCentrality:
    """The distributed job (coordinator.rs:122-135): one process per GPU; every rank holds the full counter
    array, owns a destination-row range of the CSR, and runs `run_sharded_loop`."""

    @staticmethod
    def calculate(graph, device, rank, world_size, max_iters=0, group=None, p2p=False, exchange=None, ingest="replicated"):
        """exchange: None/"nccl" = byte-max all-reduce, "p2p" (or p2p=True) = fused stores over CUDA IPC peer
        mappings, "symm" / "multicast" = fused stores over torch symmetric memory (unicast / NVSwitch multicast).
        ingest: "replicated" = `graph` is the whole edge stream on every rank; "shards" = `graph` is THIS rank's shard of it
        (host arrays) and the ranks assemble the stream in rank order with `gather_edge_shards`."""
        import time
        phase, t_prev = {}, time.perf_counter()

        def mark(name):   # wall time per phase of this rank (every phase ends in a synchronising call)
            nonlocal t_prev
            now = time.perf_counter()
            phase[name] = round((now - t_prev) * 1e3, 1)
            t_prev = now
        if ingest == "shards" and world_size > 1:
            graph = gather_edge_shards(graph, device, world_size, group)
            mark("gather_shards")
        elif ingest not in ("replicated", "shards"):
            raise ValueError(f"ingest must be 'replicated' or 'shards', not {ingest!r}")
        dg = DeviceGraph(graph, device=device, rank=rank, world_size=world_size)
        graph = None   # the gathered stream is not needed once the CSR is staged
        mark("create")
        try:
            if world_size > 1:
                if exchange in ("symm", "multicast"):
                    dg.exchange_kind = dg.enable_symmetric(group, multicast=(exchange == "multicast"))
                elif p2p or exchange == "p2p":
                    dg.enable_p2p(group)
            mark("exchange_setup")
            if world_size > 1 and getattr(dg, "p2p", False) and exchange not in ("symm", "multicast"):
                t, stats = dg.run_sharded(max_iters)          # round loop + device-side barrier behind the ABI
            else:
                t, stats = run_sharded_loop(dg, world_size, group, max_iters)
            mark("loop")
            lo, hi, c = dg.result()
            info = dg.info()
            mark("result")
            info["phase_ms"] = phase
            return HarmonicCentrality(lo, hi, c, info["n_nodes"], t, stats, info)
        finally:
            dg.close()


def _global_rank(group, r):
    import torch.distributed as dist
    return dist.get_global_rank(group, r) if group is not None else r


def _as_tensor(ptr, nbytes, dtype, dev):
    """Zero-copy torch view of a device buffer owned by the library (valid until the next step)."""
    import torch

    class _Cai:
        pass
    itemsize = torch.empty((), dtype=dtype).element_size()
    holder = _Cai()
    holder.__cuda_array_interface__ = {
        "shape": (nbytes // itemsize,), "typestr": {1: "|u1", 4: "<i4"}[itemsize], "data": (ptr, False), "version": 2}
    return torch.as_tensor(holder, device=dev)
