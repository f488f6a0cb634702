"""Several ranks of the sharded HyperBall path inside ONE emulated process: every rank is its own handle, the register
arrays and bitmaps are caller-owned numpy buffers handed over with sb200_hyperball_bind_state, and each rank's publish
targets are the other ranks' buffers by address (sb200_hyperball_set_publish_targets) -- the same calls the NVSwitch
multicast / symmetric-memory set-up makes, with unicast targets.  After every iteration every replica must equal the
oracle's registers on the rows its rank owns or reads (with the fused exchange a row is stored only into the replicas of
its subscribers; the collective exchange replicates everything).  The second half drives the same ranks through the
single-process group API (sb200_hyperball_group_link / _group_run).  Started by tests/test_hyperball_emulated.py."""
import ctypes as C
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import numpy as np  # noqa: E402
from stract_b200 import _lib, synth  # noqa: E402
L = _lib.declare(C.CDLL(os.path.join(HERE, "libsb200_emu.so")))
_lib._LIB = L
from stract_b200.webgraph import DeviceGraph, Webgraph
from stract_b200._lib import check
from oracle import DenseHyperBall, hyperball_faithful
def aligned(nbytes, dtype):
    raw = np.zeros(nbytes + 64, np.uint8); off = (-raw.ctypes.data) % 64
    return raw[off:off + nbytes].view(dtype), raw
def np_view(ptr, nbytes, dtype):
    return np.frombuffer((C.c_uint8 * nbytes).from_address(ptr), dtype=dtype)


def run(world, fused, force_mode, reuse):
    d = synth.rmat_graph(3000, 40000, seed=7)
    g = Webgraph.from_arrays(d["from_lo"], d["from_hi"], d["to_lo"], d["to_hi"], d["rel_flags"])
    hs = [DeviceGraph(g, device=0, rank=r, world_size=world) for r in range(world)]
    keep = []
    if fused:
        rb, bb = C.c_uint64(), C.c_uint64()
        check(L.sb200_hyperball_state_bytes(hs[0]._h, C.byref(rb), C.byref(bb)))
        bufs = []
        for r in range(world):
            b = [aligned(rb.value, np.uint8), aligned(rb.value, np.uint8), aligned(bb.value, np.uint32), aligned(bb.value, np.uint32)]
            bufs.append(b); keep.append(b)
            check(L.sb200_hyperball_bind_state(hs[r]._h, *(x[0].ctypes.data for x in b)))
        for r in range(world):
            peers = [p for p in range(world) if p != r]
            cols = [(C.c_uint64 * len(peers))(*(bufs[p][i][0].ctypes.data for p in peers)) for i in range(4)]
            check(L.sb200_hyperball_set_publish_targets(hs[r]._h, len(peers), *cols))
    for h in hs:
        h.set_policy(force_mode=force_mode)
    own = [h.ownership() for h in hs]
    need = [(o.astype(bool) | (((m >> r) & 1) == 1)) if fused else np.ones(len(o), bool) for r, (o, m) in enumerate(own)]
    assert np.array_equal(np.sum([o for o, _ in own], axis=0), np.ones(len(own[0][0]), np.uint8)), "every node has exactly one owner"
    if fused and world > 2:
        assert any(not n_.all() for n_ in need), "the subscriber filter should leave some rows out at world > 2"
    f = hyperball_faithful(d["from_lo"], d["from_hi"], d["to_lo"], d["to_hi"], d["rel_flags"])
    modes_seen = set()
    for rep in range(2 if reuse else 1):
        if rep:
            for h in hs: h.reset()
        ref = DenseHyperBall(d["from_lo"], d["from_hi"], d["to_lo"], d["to_hi"], d["rel_flags"])
        t = 0
        while True:
            sts = [h.step() for h in hs]
            modes_seen.update(s_["mode"] for s_ in sts)
            total = sum(s_["n_changed"] for s_ in sts)
            if not fused:   # the collective exchange: elementwise byte max over the replicas (what the NCCL MAX all-reduce does)
                ptrs = [h.exchange_ptrs() for h in hs]
                regs = [np_view(p[0], p[1], np.uint8) for p in ptrs]; fr = [np_view(p[2], p[3], np.uint8) for p in ptrs]
                mr = np.maximum.reduce(regs); mf = np.maximum.reduce(fr)
                for x in regs: x[:] = mr
                for x in fr: x[:] = mf
            for h in hs: h.exchange_done(total)
            ch = ref.step(); t += 1
            regs = [h.registers() for h in hs]
            want = ref.registers()
            for r in range(world):
                assert np.array_equal(regs[r][need[r]], want[need[r]]), ("replica differs from the oracle on a row it owns or reads", world, r, fused, force_mode, t)
            assert (total == 0) == (not ch), (t, total, ch)
            if total == 0: break
        res = [h.result() for h in hs]
        lo = np.concatenate([r[0] for r in res]); hi = np.concatenate([r[1] for r in res]); c = np.concatenate([r[2] for r in res])
        key = hi.astype(object) * (1 << 64) + lo.astype(object); o = np.argsort(key)
        assert np.array_equal(lo[o], f["ids_lo"]) and np.array_equal(c[o], f["centrality"]) and t == f["iters"], (world, fused, force_mode, rep)
    for h in hs: h.close()
    print("world", world, "fused" if fused else "collective", "force_mode", force_mode, "reuse", reuse, "modes", sorted(modes_seen), "ok", flush=True)
    return modes_seen


def run_group(world, force_mode, options=None):
    """The round loop behind the ABI, single-process form: link + run, then the union of the owned results."""
    from stract_b200.webgraph import DeviceGroup
    d = synth.rmat_graph(3000, 40000, seed=7)
    g = Webgraph.from_arrays(d["from_lo"], d["from_hi"], d["to_lo"], d["to_hi"], d["rel_flags"])
    f = hyperball_faithful(d["from_lo"], d["from_hi"], d["to_lo"], d["to_hi"], d["rel_flags"])
    grp = DeviceGroup(g, [0] * world)
    for h in grp.ranks:
        h.set_policy(force_mode=force_mode)
    for rep in range(2):
        if rep:
            grp.reset()
            for h in grp.ranks:                     # the tuning switches may change between computations of one handle
                for k, v in (options or {}).items():
                    h.set_option(k, v)
        t, stats = grp.run()
        lo, hi, c = grp.result()
        assert t == f["iters"] and np.array_equal(lo, f["ids_lo"]) and np.array_equal(hi, f["ids_hi"]) and np.array_equal(c, f["centrality"]), (world, force_mode, rep)
    grp.close()
    print("group world", world, "force_mode", force_mode, "options", options, "ok", flush=True)


for world in (2, 4, 8):
    run_group(world, -1)
run_group(3, 2)
run_group(4, -1, {"quad_side_ctas": 0, "publish_all": 1, "owned_items": 0})
run_group(3, -1, {"quad_side_ctas": 4, "publish_all": 0, "owned_items": 1})
for world in (2, 3):
    for fused in (True, False):
        run(world, fused, -1, False)
        run(world, fused, 2, False)                 # push on every iteration, owned-row source-major CSR
        m = run(world, fused, -1, True)             # the policy builds it lazily on the second run and switches to push
        assert 2 in m, m
print("sharded emulated parity ok")
