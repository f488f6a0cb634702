"""The betweenness oracles, no GPU: the canonical-order restatement (betweenness_oracle_mt.cpp) pinned on the reference's
`path` test (betweenness.rs:203-218) and checked against the literal transcription of `calculate` -- exactly where no node
has two successors on a shortest-path DAG, within 1e-12 relative where the pinned summation order reassociates the sums."""
import math

import numpy as np
import pytest

import betweenness_oracle as B


def _canonical_map(n, fr, tr, sources):
    cent, reached, md = B.canonical(n, fr, tr, sources, threads=3)
    return B.as_map(cent, reached), md


def _bits(x):
    return np.float64(x).view(np.uint64)


def _same(a, b):
    return a.keys() == b.keys() and all((math.isnan(a[k]) and math.isnan(b[k])) or _bits(a[k]) == _bits(b[k]) for k in a)


def test_path_known_answer():
    n, fr, tr = B.path(5)
    got, md = _canonical_map(n, fr, tr, range(5))
    assert got == {0: 0.0, 1: 0.15, 2: 0.2, 3: 0.15, 4: 0.0} and md == 4
    lit, lmd = B.literal(n, fr, tr, range(5))
    assert _same(got, lit) and lmd == 4
    # the reference iterates a hash set: the source order does not change a sum of one term per node
    got2, _ = _canonical_map(n, fr, tr, [3, 1, 4, 0, 2])
    assert got2 == got


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_literal_equals_canonical_on_trees(seed):
    n, fr, tr = B.random_tree(300, seed)
    rng = np.random.default_rng(seed)
    src = rng.permutation(n)[:120]
    got, md = _canonical_map(n, fr, tr, src)
    lit, lmd = B.literal(n, fr, tr, src)
    assert _same(got, lit) and md == lmd


@pytest.mark.parametrize("seed,n,m", [(4, 200, 900), (5, 400, 1200), (6, 60, 1500)])
def test_literal_within_1e12_of_canonical(seed, n, m):
    n, fr, tr = B.random_graph(n, m, seed)
    src = np.random.default_rng(seed).permutation(n)[: n // 2]
    got, md = _canonical_map(n, fr, tr, src)
    lit, lmd = B.literal(n, fr, tr, src)
    assert got.keys() == lit.keys() and md == lmd
    a = np.array([got[k] for k in sorted(got)]); b = np.array([lit[k] for k in sorted(lit)])
    assert np.all(np.abs(a - b) <= 1e-12 * np.abs(b))
    assert np.count_nonzero(a) > n // 4


def test_no_and_one_source():
    n, fr, tr = B.path(5)
    assert _canonical_map(n, fr, tr, []) == ({}, 0)
    assert B.literal(n, fr, tr, []) == ({}, 0)
    # n == 1: norm = 1 * 0 = 0; 0/0 is NaN, x/0 is +inf
    got, md = _canonical_map(n, fr, tr, [1])
    lit, lmd = B.literal(n, fr, tr, [1])
    assert _same(got, lit) and md == lmd == 3
    assert set(got) == {1, 2, 3, 4}
    assert math.isnan(got[1]) and math.isnan(got[4]) and got[2] == math.inf and got[3] == math.inf


@pytest.mark.parametrize("k,last_pred", [(31, -0.25), (32, -math.inf)])
def test_diamond_chain_wraps_i32(k, last_pred):
    n, fr, tr = B.diamonds(k)
    sink = 3 * k
    for src in ([0, sink], [0, 3, 1, 4, 2]):
        got, md = _canonical_map(n, fr, tr, src)
        lit, lmd = B.literal(n, fr, tr, src)
        assert md == lmd == 2 * k
        assert _same(got, lit)
    # from m_0: sigma[a_{k-1}] = 2^(k-1) over sigma[m_k] = 2^k, which the i32 wraps to -2^31 (k = 31) or to 0 (k = 32);
    # with the sources [m_0, m_k] (m_k reaches nothing) the norm is 2
    got, _ = _canonical_map(n, fr, tr, [0, sink])
    assert got[sink - 2] == last_pred and got[sink - 1] == last_pred


def test_disconnected_parts():
    # two paths and an isolated pair; sources in both parts and one that reaches nothing
    n = 12
    fr = np.array([0, 1, 2, 3, 5, 6, 7, 9], np.uint32); tr = np.array([1, 2, 3, 4, 6, 7, 8, 10], np.uint32)
    src = [4, 0, 5, 6, 11]
    got, md = _canonical_map(n, fr, tr, src)
    lit, lmd = B.literal(n, fr, tr, src)
    assert _same(got, lit) and md == lmd == 4
    assert set(got) == {0, 1, 2, 3, 4, 5, 6, 7, 8, 11}       # 9, 10 are reached by no source
    norm = 5.0 * 4.0
    assert got[1] == 3.0 / norm and got[7] == (1.0 + 1.0) / norm and got[6] == 2.0 / norm and got[11] == 0.0


def test_self_loops_and_repeats_change_nothing():
    n, fr, tr = B.random_graph(80, 400, 9, self_loops=False)
    src = np.arange(0, 80, 3)
    base, md = _canonical_map(n, fr, tr, src)
    fr2 = np.concatenate([fr, fr[:50], np.arange(0, 80, 2, dtype=np.uint32)])
    tr2 = np.concatenate([tr, tr[:50], np.arange(0, 80, 2, dtype=np.uint32)])
    got, md2 = _canonical_map(n, fr2, tr2, src)
    assert _same(got, base) and md == md2
    lit, _ = B.literal(n, fr2, tr2, src)
    assert got.keys() == lit.keys()


def test_threads_do_not_change_bits():
    n, fr, tr = B.random_graph(500, 3000, 11)
    src = np.random.default_rng(0).permutation(n)[:333]
    a = B.canonical(n, fr, tr, src, threads=1)
    b = B.canonical(n, fr, tr, src, threads=7)
    assert B.same_bits(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]
