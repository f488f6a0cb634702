"""world_size-2 `gloo` test of the multi-rank host logic (stract_b200.webgraph.run_sharded_loop): interleaved
row ownership, byte-max all-reduce of the register replicas and changed bitmaps, changed-count all-reduce and the
termination rule.  The per-rank compute engine is a numpy stand-in (tests only); on the GPU box the same
loop drives the CUDA DeviceGraph (tests/test_sharded_gpu.py)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import DenseHyperBall
from stract_b200 import synth


class NumpyShard:
    """Owns the destination rows of its interleaved 32-row blocks; the full register array is replicated."""

    def __init__(self, d, rank, world):
        self.orc = DenseHyperBall(d["from_lo"], d["from_hi"], d["to_lo"], d["to_hi"], d["rel_flags"])
        n = self.orc.n_nodes
        self.n = n
        lo, hi = self.orc.ids()
        # rebuild (to, from) rank pairs the same way the oracle does
        ids = (hi.astype(object) << 64) | lo.astype(object)
        pos = {int(v): i for i, v in enumerate(ids)}
        f = [pos[(int(h) << 64) | int(l)] for l, h in zip(d["from_lo"], d["from_hi"])]
        t = [pos[(int(h) << 64) | int(l)] for l, h in zip(d["to_lo"], d["to_hi"])]
        seen, edges = set(), []
        skipmask = 0x6FED00
        for a, b_, r in zip(f, t, d["rel_flags"]):
            if (a, b_) in seen:
                continue
            seen.add((a, b_))
            if int(r) & skipmask:
                continue
            edges.append((a, b_))
        self.edges = np.array(edges, np.int64).reshape(-1, 2)
        # interleaved ownership: 32-row block b belongs to rank b % world (as in the CUDA library)
        self.own = ((np.arange(n) >> 5) % world) == rank
        self.regs = torch.from_numpy(self.orc.registers().reshape(-1).copy())
        self.front = torch.zeros((n + 31) // 32, dtype=torch.int32)
        self.changed_prev = np.ones(n, bool)

    def step(self):
        old = self.regs.numpy().reshape(self.n, 64).copy()
        new = old.copy()
        m = self.changed_prev[self.edges[:, 0]] & self.own[self.edges[:, 1]]
        src, dst = self.edges[m, 0], self.edges[m, 1]
        np.maximum.at(new, dst, old[src])
        ch = (new != old).any(1)
        self.regs.numpy().reshape(self.n, 64)[self.own] = new[self.own]
        bits = np.zeros(((self.n + 31) // 32) * 32, np.uint8)
        bits[:self.n][self.own] = ch[self.own]
        words = np.packbits(bits.reshape(-1, 32), axis=1, bitorder="little").view(np.uint32).reshape(-1).astype(np.int64)
        self.front.copy_(torch.from_numpy(words.astype(np.uint32).view(np.int32)))
        return {"n_changed": int(ch[self.own].sum())}

    def exchange_tensors(self):
        return self.regs, self.front

    def exchange_done(self, total):
        w = self.front.numpy().view(np.uint32)
        bits = np.unpackbits(w.view(np.uint8).reshape(-1, 4), axis=1, bitorder="little").reshape(-1)[:self.n]
        self.changed_prev = bits.astype(bool)


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from stract_b200.webgraph import run_sharded_loop
        d = synth.uniform_graph(700, 2500, 5)
        eng = NumpyShard(d, rank, world)
        t, stats = run_sharded_loop(eng, world)
        ref = DenseHyperBall(d["from_lo"], d["from_hi"], d["to_lo"], d["to_hi"], d["rel_flags"])
        it = ref.run()
        ok = np.array_equal(eng.regs.numpy().reshape(-1, 64), ref.registers()) and t == it
        ok = ok and stats[-1]["n_changed_global"] == 0 and all(s["n_changed_global"] > 0 for s in stats[:-1])
        q.put((rank, bool(ok), t, it))
    finally:
        dist.destroy_process_group()


def test_two_rank_exchange_protocol_gloo():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok, _, _ in res), res


def _gather_worker(rank, world, port, q, counts):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from stract_b200.webgraph import Webgraph, gather_edge_shards, shard_bounds
        total = sum(counts)
        rng = np.random.default_rng(11)
        cols = [rng.integers(0, 2 ** 63, total, dtype=np.uint64) * np.uint64(2) + np.uint64(1) for _ in range(5)]   # top bit set too
        lo = sum(counts[:rank]); hi = lo + counts[rank]
        if rank % 2:   # numpy and torch shards both
            shard = Webgraph.from_arrays(*[torch.from_numpy(c[lo:hi].view(np.int64).copy()) for c in cols])
        else:
            shard = Webgraph.from_arrays(*[c[lo:hi].copy() for c in cols])
        full = gather_edge_shards(shard, "cpu", world)
        ok = full.n_edges == total
        for got, want in zip((full.from_lo, full.from_hi, full.to_lo, full.to_hi, full.rel), cols):
            ok = ok and np.array_equal(got.numpy().view(np.uint64), want)
        b = [shard_bounds(total, r, world) for r in range(world)]
        ok = ok and b[0][0] == 0 and b[-1][1] == total and all(b[i][1] == b[i + 1][0] for i in range(world - 1))
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("counts", [[1000, 1000, 1000], [1000, 1000, 37], [334, 334, 332], [500, 0, 200], [0, 0, 0], [7, 0, 0]])
def test_edge_shards_gathered_in_rank_order_gloo(counts):
    """`gather_edge_shards`: equal shards (in-place prefix), a short or empty trailing shard, ragged shards (re-packed) and
    an empty stream all give every rank the concatenation of the shards in rank order."""
    world = len(counts)
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gather_worker, args=(r, world, port, q, counts)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok in res), res
