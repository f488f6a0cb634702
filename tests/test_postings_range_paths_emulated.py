"""The checks of tests/test_postings_range_paths_gpu.py on the CPU SIMT emulator (tests/emu), reduced: fewer queries,
slops and k, and the near-limit positional index at max_doc = 2^25 - 2 instead of 2^31 - 2.  The fixtures are the same
(position widths 0..32, positions from 2^31 up, 5-byte VInt deltas, the u32 slop wrap, the tf 2^16 + 1 posting, doc ids
up to max_doc - 1, range fields with tfs up to 2^32 - 1 next to the positional fields); the term beyond 4 GiB of
positions runs on the GPU only."""
import numpy as np
import pytest

import test_postings_range_paths_gpu as P
from test_bm25_emulated import emulated  # noqa: F401  (the fixture that swaps in the emulated library)

REDUCED_LIMIT = (1 << 25) - 2


def test_phrases_and_patterns(emulated, monkeypatch):
    fx = P.make(61, P.MEDIUM)
    assert P.check_phrases(fx, np.random.default_rng(1), 6, slops=(0, 3), ks=(4096,), python_rows=6) > 0
    P.check_patterns(fx)
    fx["seg"].close()


@pytest.fixture(scope="module")
def fields(emulated):
    return P.make_fields(81, P.MEDIUM, big=False)


def test_multi_field_optic_plans(fields, monkeypatch):
    P.check_multi_field(fields, np.random.default_rng(11), 4, ks=(100,))
    P.check_optic(fields, np.random.default_rng(12), 4)
    P.check_plans(fields, np.random.default_rng(13), 8, monkeypatch=monkeypatch)


def test_recall_webpages(fields):
    P.check_webpages(fields, np.random.default_rng(14), 4)


def test_reduced_near_limit_positional_index(emulated):
    fx = P.make(91, REDUCED_LIMIT, counts=False)
    P.check_phrases(fx, np.random.default_rng(15), 4, slops=(0, 3), ks=(4096,), python_rows=5)
    P.check_patterns(fx, anchors=False)
    fx["seg"].close()
