"""BM25 CUDA kernels on a CPU SIMT emulator (tests/emu): the unmodified stract_b200/csrc/bm25*.cu{,h} sources are
compiled by g++ against a shim in which every CUDA thread is a coroutine, warps meet at every *_sync intrinsic and
blocks at __syncthreads().  Lanes run one after the other between two barriers -- the largest skew a real GPU may
show -- so shared-memory races that converged execution hides turn into wrong answers here (this is how the
fill-level race in k_topk_warp was found).  The parity functions are the ones of tests/test_bm25_gpu.py, run against
the oracle exactly as on the GPU; this file only swaps the library underneath them.

What this is NOT: a performance statement, a memory-model checker, or part of the product -- stract_b200 never loads
the emulator; only this test does.  It lets kernels written without a GPU at hand, as bm25_and3.cuh and bm25_or3.cuh
were, be checked bit-exactly before their first GPU run."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")


@pytest.fixture(scope="module")
def emulated():
    subprocess.check_call(["make", "-C", EMU], stdout=subprocess.DEVNULL)
    from stract_b200 import _lib
    L = _lib.declare(C.CDLL(os.path.join(EMU, "libsb200_emu.so")))
    assert b"emulation" in L.sb200_version()
    saved = _lib._LIB
    _lib._LIB = L
    import test_bm25_gpu as T   # the GPU parity tests, reused as plain functions
    try:
        yield T
    finally:
        _lib._LIB = saved


def test_default_kernels_against_oracle(emulated):
    T = emulated
    T.test_droopy_tax_kat()
    T.test_and_queries_bit_exact()
    T.test_or_queries_bit_exact_up_to_two_terms()
    T.test_or_three_plus_terms_canonical_order()
    T.test_ties_order_by_doc_and_padding()
    T.test_signal_combine_bit_exact()
    import test_round1_late_gpu as late
    late.test_positions_record_option_skip_entries()
    late.test_term_info_store_decoded_on_device()
    late.test_searcher_over_three_segments_matches_one_big_segment()
    late.test_signal_searcher_over_segments_matches_one_big_segment()
    T.test_malformed_postings_rejected()
    import test_golden
    test_golden.check_path2_against_golden()   # committed fixtures, no oracle call


def test_unit_based_and_kernel_against_oracle(emulated, monkeypatch):
    emulated.test_and3_unit_kernel_bit_exact(monkeypatch)


def test_union_kernel_against_oracle(emulated):
    """A reduced form of test_or3_union_kernel_bit_exact (the full one takes ~10 min emulated): OR with 1..8 clauses,
    absent clauses, doc-range items + merge, signal combine with 4 / 2 / 0 columns."""
    emulated.union_kernel_against_oracle(33, 60_000, [1, 5, 127, 128, 129, 300, 1000, 1280, 5000, 12000, 20000],
                                         nq=24, ks=(1, 100), pad_every=5, sig_nq=16, sig_k=200)


def test_multi_field_signals_against_oracle(emulated):
    import test_multi_signal_gpu as M
    M.test_multi_field_signals_bit_exact()
    M.test_optic_rule_boosts_bit_exact()
    M.test_all_numeric_signals_from_raw_columns_in_the_program()
    M.test_signal_compute_order_mirror()
    M.test_coefficient_precedence_mirror()


def test_block_wand_replay_against_oracle(emulated):
    emulated.test_or_wand_replay_matches_block_wand_bit_for_bit()


def test_packed_result_copy(emulated, monkeypatch):
    emulated.test_packed_result_copy_equals_dense(monkeypatch)


def test_numeric_signal_transforms_against_oracle(emulated):
    import test_numeric_signals_gpu as N
    N.test_every_numeric_signal_bit_exact(N.NOW, ([120, None, 30, 0, 77, 1, 5], 233), 2)
    N.test_every_numeric_signal_bit_exact(None, None, None)
    N.test_subset_of_signals_in_enum_order()
