"""The checks of tests/test_graph_range_gpu.py on the CPU SIMT emulator (tests/emu), reduced: the range graph at 2^15 - 1
nodes with a hub of 11 900 in-edges and a 12 000-edge push source instead of 2^17 - 1 / 70 000 / 70 000.  Every boundary
stays: rows of exactly 1 .. 16 385 in-edges, rows of 9 and 17 work items, 48 multi-item rows, 64 search bits, 65 and
129 similarity targets and the 300-node chain with its 254-level cap.  HyperBall runs the default policy (fresh and reset)
and the group at 3 ranks; the forced modes and 2 ranks run on the GPU."""
import numpy as np
import pytest

import graph_range as G
import test_graph_range_gpu as T
from stract_b200.webgraph import SKIPPED_REL
from test_bm25_emulated import emulated  # noqa: F401  (the fixture that swaps in the emulated library)


@pytest.fixture(scope="module")
def reduced():
    return G.range_graph(1, "reduced")


def test_hyperball_stepwise(emulated, reduced):
    # the default policy, fresh and on a reset handle (seed pulls, merges, dense and frontier pulls, then pushes); the
    # forced modes run on the GPU
    T.check_hyperball_stepwise(reduced, modes=(-1,))


def test_sharded_group(emulated, reduced):
    T.check_sharded_group(reduced, worlds=(3,), modes=(-1,))


def test_long_run_chain(emulated):
    T.check_long_run(G.chain_graph(300))


@pytest.mark.parametrize("mask", [0, SKIPPED_REL])
def test_distances(emulated, reduced, mask):
    T.check_range_distances(reduced, mask)


def test_distances_chain(emulated):
    T.check_chain_distances(G.chain_graph(300), 0)


def test_approx_harmonic(emulated, reduced):
    T.check_approx_harmonic(reduced, 0, max_dists=(1, 253))
    T.check_approx_harmonic(G.chain_graph(300), 0, sizes=(1, 65), max_dists=(253,), big_num_nodes=(65,))


def test_inbound_similarity(emulated, reduced):
    T.check_inbound_similarity(reduced, 0, np.random.default_rng(9))
