"""Iteration 0 of HyperBall from the 2-byte seeds (the SEED pull variants) against the CPU oracle.  Needs a GPU;
tests/test_seed_iteration_emulated.py runs the same functions on the CPU SIMT emulator.

After a reset every counter has one non-zero register, so the first pull reads a 2-B seed per source instead of the
64-B row.  These tests check that the result is the oracle's bit for bit: for seeds with every register index, for
reused and caller-bound state, and for the replicas of a sharded group."""
import ctypes as C

import numpy as np
import pytest

from oracle import DenseHyperBall, hyperball_faithful
from stract_b200 import _lib, synth
from stract_b200._lib import check
from stract_b200.webgraph import DeviceGraph, DeviceGroup, Webgraph

pytestmark = pytest.mark.gpu
M64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15   # FastHasher's multiplier: the register index of a counter is (id_lo * GOLDEN) >> 58


def _args(d):
    return (d["from_lo"], d["from_hi"], d["to_lo"], d["to_hi"], d["rel_flags"])


def _graph(d):
    return Webgraph.from_arrays(*_args(d))


def _all_register_ids():
    """Low id halves whose seeds hit every register index 0..63, starting with 0 (hash 0: index 0, value 65)."""
    seen, ids, x = set(), [], 0
    while len(seen) < 64:
        j = ((x * GOLDEN) & M64) >> 58
        if x == 0 or j not in seen:
            ids.append(x)
            seen.add(j)
        x += 1
    return ids


def _seed_graph():
    """Every node is a source and a destination; rows of every class: short (quad), long (warp), and one longer than
    a 1024-edge work item (merge)."""
    rng = np.random.default_rng(11)
    lo_ids = _all_register_ids()
    lo_ids += list(range(1000, 1000 + 400 - len(lo_ids)))
    n = len(lo_ids)
    f = list(range(n)) + list(rng.integers(0, n, 3000)) + list(rng.integers(0, n, 1500)) + list(rng.integers(0, n, 200))
    t = [(i + 1) % n for i in range(n)] + list(rng.integers(0, n, 3000)) + [0] * 1500 + [5] * 200
    lo = np.array(lo_ids, np.uint64)
    fi, ti = np.array(f), np.array(t)
    hi = np.uint64(7)
    k = len(f)
    return dict(from_lo=lo[fi], from_hi=np.full(k, hi, np.uint64), to_lo=lo[ti], to_hi=np.full(k, hi, np.uint64),
                rel_flags=np.zeros(k, np.uint64))


def _check_iteration0(dg, orc):
    st = dg.step()
    assert st["t"] == 0 and st["n_changed"] == orc.step()
    assert np.array_equal(dg.registers(), orc.registers()), "registers differ after iteration 0"
    s, e = dg.kahan()
    os_, oe = orc.kahan()
    assert np.array_equal(s, os_) and np.array_equal(e, oe), "KahanSum differs after iteration 0"


def _check_rest(dg, d):
    dg.run()
    lo, hi, c = dg.result()
    ref = hyperball_faithful(*_args(d))
    assert np.array_equal(lo, ref["ids_lo"]) and np.array_equal(hi, ref["ids_hi"]) and np.array_equal(c, ref["centrality"])


@pytest.mark.parametrize("force_mode", [-1, 1, 2])
def test_iteration0_every_register_index(force_mode):
    d = _seed_graph()
    lo = set(int(x) for x in d["to_lo"])
    assert 0 in lo and len({((x * GOLDEN) & M64) >> 58 for x in lo}) == 64
    orc = DenseHyperBall(*_args(d), threads=4)
    dg = DeviceGraph(_graph(d))
    try:
        dg.set_policy(force_mode=force_mode)
        assert np.array_equal(dg.registers(), orc.registers())
        assert dg.registers().max() == 65   # id_lo = 0
        _check_iteration0(dg, orc)
        _check_rest(dg, d)
    finally:
        dg.close()
        orc.close()


def test_profile_seed_families_only_in_iteration0():
    d = synth.rmat_graph(3000, 40_000, seed=7)
    dg = DeviceGraph(_graph(d))
    try:
        dg.set_profiling(True)
        iters, stats = dg.run()
        prof = {p["name"]: p for p in dg.profile()}
        dense_later = sum(1 for s in stats if s["t"] >= 1 and s["mode"] == 0)
        assert stats[0]["mode"] == 0 and dense_later >= 1
        for fam in ("warp", "quad"):
            seed, dense = prof[f"k_pull_{fam}<seed>"], prof[f"k_pull_{fam}<dense>"]
            assert seed["launches"] == 1 and seed["alg_bytes"] > 0, (fam, seed)
            assert dense["launches"] == dense_later, (fam, dense, stats)
    finally:
        dg.close()


def test_reused_handle_with_forward_csr():
    d = synth.rmat_graph(3000, 40_000, seed=7)
    dg = DeviceGraph(_graph(d))
    try:
        dg.run()
        dg.reset()
        _, stats = dg.run()   # a reused handle builds the source-major CSR and pushes late iterations
        assert any(s["mode"] == 2 for s in stats)
        dg.reset()
        orc = DenseHyperBall(*_args(d), threads=4)
        try:
            _check_iteration0(dg, orc)
        finally:
            orc.close()
        _check_rest(dg, d)
    finally:
        dg.close()


def _device_buffer(nbytes, keep):
    """64-B aligned device memory for sb200_hyperball_bind_state (host memory on the emulator, which has one address space)."""
    if b"emulation" in _lib.lib().sb200_version():
        raw = np.zeros(nbytes + 64, np.uint8)
        ptr = raw.ctypes.data
    else:
        import torch
        raw = torch.zeros(nbytes + 64, dtype=torch.uint8, device="cuda")
        ptr = raw.data_ptr()
    keep.append(raw)
    return ptr + (-ptr) % 64


def test_bound_state():
    d = synth.rmat_graph(3000, 40_000, seed=7)
    dg = DeviceGraph(_graph(d))
    keep = []
    try:
        L = _lib.lib()
        rb, bb = C.c_uint64(), C.c_uint64()
        check(L.sb200_hyperball_state_bytes(dg._h, C.byref(rb), C.byref(bb)))
        ptrs = [_device_buffer(n, keep) for n in (rb.value, rb.value, bb.value, bb.value)]
        check(L.sb200_hyperball_bind_state(dg._h, *ptrs))
        orc = DenseHyperBall(*_args(d), threads=4)
        try:
            assert np.array_equal(dg.registers(), orc.registers())
            _check_iteration0(dg, orc)
        finally:
            orc.close()
        _check_rest(dg, d)
    finally:
        dg.close()


@pytest.mark.parametrize("world", [2, 4])
def test_group_replicas_after_iteration0(world):
    d = synth.rmat_graph(3000, 40_000, seed=7)
    grp = DeviceGroup(_graph(d), [0] * world)
    orc = DenseHyperBall(*_args(d), threads=4)
    try:
        own = [h.ownership() for h in grp.ranks]
        need = [o.astype(bool) | (((m >> r) & 1) == 1) for r, (o, m) in enumerate(own)]
        t, _ = grp.run(max_iters=1)
        assert t == 1
        orc.step()
        want = orc.registers()
        for r, h in enumerate(grp.ranks):   # every replica is right on the rows its rank owns or reads
            got = h.registers()
            assert np.array_equal(got[need[r]], want[need[r]]), r
        grp.run()
        lo, hi, c = grp.result()
        ref = hyperball_faithful(*_args(d))
        assert np.array_equal(lo, ref["ids_lo"]) and np.array_equal(hi, ref["ids_hi"]) and np.array_equal(c, ref["centrality"])
    finally:
        orc.close()
        grp.close()
