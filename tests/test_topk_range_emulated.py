"""The top-k range checks of tests/test_topk_range_gpu.py on the CPU SIMT emulator (tests/emu), reduced: fewer k values
(still one on each side of every buffer rule's power of two), and the split batches at max_doc = 2^18 with W = 4 and W = 2
(W = 16 takes 16 * 32768 postings in one query, GPU only)."""
import numpy as np

import test_topk_range_gpu as G
import topk_range as R
from test_bm25_emulated import emulated  # noqa: F401  (the fixture that swaps in the emulated library)

KS = [1, 32, 33, 992, 993, 1024, 1025, 3072, 3073, 4064, 4065, 4096]
MAX_DOC = 40_000


def test_boundary_k(emulated):
    fx = G.make_tie(61, MAX_DOC, KS)
    G.check_boundary_k(fx, KS)
    G.check_k_refused(fx)
    G.check_signals(fx, [1, 33, 1025, 3073], R.special_columns(MAX_DOC, 7), max_docs_list=(0, 137))
    G.check_multi(fx, [1, 1025, 3072, 3073], R.special_columns(MAX_DOC, 8), slot_counts=(8, 16))


def test_multi_field_buffer_lands_on_cap(emulated):
    G.check_landing(max_doc=40_000, k=1024, ns=8)


def test_split_batches(emulated):
    fx = G.make_split(71, 1 << 18, [4 * 32768 - 2048, G.W2_DF])
    G.check_split(fx, [(0, 1, 4), (0, 4096, 4), (1, 10, 2)])


def test_optic_plan_webpages_segments(emulated):
    fx = G.make_tie(61, MAX_DOC, KS)
    cols = R.special_columns(MAX_DOC, 8)
    G.check_optic(fx, [1, 1025, 4096], cols)
    G.check_plan(fx, [1, 992, 993, 4064, 4065], cols)
    G.check_webpages(fx, [33, 1025], cols)
    G.check_segments(fx, [1, 33, 1025, 4096], R.special_columns(MAX_DOC, 7))


def test_phrases_boundary_k(emulated):
    G.check_phrases_k([1, 32, 33, 1024, 1025, 4096], 4)
