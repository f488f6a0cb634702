"""The posting-range checks of tests/test_postings_range_gpu.py on the CPU SIMT emulator (tests/emu), reduced: fewer
queries, and the large index at max_doc = 2^25 - 2 instead of 2^31 - 2 (doc deltas up to 25 bits and 4-byte VInt gaps;
the 31-bit deltas and 5-byte gaps run on the GPU only).  Tf widths 0..32, 5-byte VInt tfs, block-wand code 255 and every
fieldnorm code are the same as on the GPU."""
import numpy as np

import test_postings_range_gpu as P
from test_bm25_emulated import emulated  # noqa: F401  (the fixture that swaps in the emulated library)

REDUCED_LIMIT = (1 << 25) - 2


def test_medium_index(emulated, monkeypatch):
    fx = P.make(41, P.MEDIUM)
    rng = np.random.default_rng(1)
    P.check_single_term_raw(fx)
    P.check_and(fx, rng, 24, ks=(10, P.MAX_K), monkeypatch=monkeypatch)
    P.check_or(fx, rng, 8, (10, 1000), 6, 200, sig_cols=(2,))
    P.check_wand(fx, rng, 3, ks=(10,))
    P.check_docsets(fx)


def test_medium_index_record_option_2(emulated):
    fx = P.make(43, P.MEDIUM, record_option=2)
    rng = np.random.default_rng(4)
    P.check_single_term_raw(fx, ks=(P.MAX_K,))
    P.check_and(fx, rng, 12, ks=(P.MAX_K,))
    P.check_or(fx, rng, 4, (1000,), 0, 0, sig_cols=())
    P.check_wand(fx, rng, 2, ks=(10,))


def test_reduced_near_limit_index(emulated):
    fx = P.make(47, REDUCED_LIMIT)
    assert 24 in fx["produced"]["wd"] and 4 in fx["produced"]["gap_bytes"]
    rng = np.random.default_rng(5)
    P.check_single_term_raw(fx, ks=(P.MAX_K,))
    P.check_and(fx, rng, 12, ks=(P.MAX_K,))
    P.check_or(fx, rng, 4, (1000,), 0, 0, sig_cols=())
    P.check_wand(fx, rng, 2, ks=(10,))
    P.check_docsets(fx)


def test_max_doc_limit_refused(emulated):
    P.check_max_doc_limit()


def test_positions_read_back(emulated):
    P.check_positions()
