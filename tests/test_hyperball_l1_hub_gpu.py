"""The L1 budget of the pulls' hub sources (the handle option "l1_hub_kb") changes where gathers are cached, never what is
computed: under each kernel family, from the seed iteration on, the registers and KahanSums after every iteration are the
oracle's, bit for bit, for every budget.  Needs a GPU; test_hyperball_l1_hub_emulated.py runs the same functions on the
CPU SIMT emulator."""
import math

import numpy as np
import pytest

from oracle import DenseHyperBall
from stract_b200 import synth
from stract_b200.webgraph import DeviceGraph, Webgraph

pytestmark = pytest.mark.gpu

N_NODES, N_EDGES = 3000, 40000
# rows gathered through L1 = kb * 1024 / 64.  2.5 KB puts the boundary at row 40, inside the node range: the 32 sources of a
# long row's gather batch and the 4 of a short row's quad step fall on both sides of it, and so do the destination rows
# themselves.  None: the handle's default, never set.
BUDGETS = (None, 0, 2.5)


def _args(d):
    return (d["from_lo"], d["from_hi"], d["to_lo"], d["to_hi"], d["rel_flags"])


def _graph():
    # long rows split over several work items next to short rows and rows without in-edges
    return synth.rmat_graph(N_NODES, N_EDGES, seed=17)


def _oracle_iterations(d):
    orc = DenseHyperBall(*_args(d), threads=4)
    out = []
    while True:
        n = orc.step()
        out.append((n, orc.registers(), *orc.kahan()))
        if n == 0:
            return orc.n_nodes, out


def _check(force_mode):
    d = _graph()
    n_nodes, ref = _oracle_iterations(d)
    every_row = math.ceil(n_nodes * 64 / 1024)   # every gather through L1, as without the split
    dg = DeviceGraph(Webgraph.from_arrays(*_args(d)))
    try:
        dg.set_policy(force_mode=force_mode)
        for kb in BUDGETS + (every_row, 0):   # one computation per budget on the same handle
            if kb is not None:
                dg.set_option("l1_hub_kb", kb)
            dg.reset()
            for t, (n, regs, ks, ke) in enumerate(ref):
                st = dg.step()
                assert st["t"] == t and st["n_changed"] == n, (kb, t)
                assert np.array_equal(dg.registers(), regs), f"registers differ in iteration {t} with {kb} KB"
                s, e = dg.kahan()
                assert np.array_equal(s, ks) and np.array_equal(e, ke), f"KahanSum differs in iteration {t} with {kb} KB"
    finally:
        dg.close()


@pytest.mark.parametrize("force_mode", [0, 1, 2])
def test_l1_hub_budgets_match_oracle_every_iteration(force_mode):
    _check(force_mode)


def test_l1_hub_option_range():
    d = synth.rmat_graph(200, 800, seed=18)
    dg = DeviceGraph(Webgraph.from_arrays(*_args(d)))
    try:
        for bad in (-1, -0.5, float("nan"), 2.0 ** 30 + 1):
            with pytest.raises(Exception):
                dg.set_option("l1_hub_kb", bad)
        for good in (0, 0.0625, 2.0 ** 30):
            dg.set_option("l1_hub_kb", good)
    finally:
        dg.close()
