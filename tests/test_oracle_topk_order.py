"""The oracle's f64 top-k order (TopN<double>, oracle/oracle_postings.cpp) on hand-made lists: f64::total_cmp over the bits,
-0.0 below +0.0, -inf / +inf at the ends, every NaN tied below -inf (the library's NaN rule, DESIGN §5), doc ascending on
equal keys, in the final sort and in the threshold test of the truncating buffer."""
import numpy as np

import oracle
import topk_range as R

VALUES = [0.0, -0.0, -np.inf, np.inf, R.NAN_P, R.NAN_N, -1.5, 2.0, R.SUB, -R.SUB, R.F64_MAX, -R.F64_MAX]


def test_total_cmp_order_of_special_values():
    totals = np.array(VALUES, np.float64)
    docs = np.arange(totals.size, dtype=np.uint32)[::-1].copy()
    od, ot = oracle.topn_f64(totals, docs, totals.size)
    order = [np.inf, R.F64_MAX, 2.0, R.SUB, 0.0, -0.0, -R.SUB, -1.5, -R.F64_MAX, -np.inf]
    assert np.array_equal(R.bits(ot[:10]), R.bits(order))
    assert np.isnan(ot[10:]).all() and list(od[10:]) == sorted(od[10:])   # the two NaNs tie: doc ascending
    assert od.tolist() == R.expected_topk(totals, docs, totals.size)[0].tolist()


def test_ties_and_truncation_against_restatement():
    """many pushes with every special value repeated: the buffer truncates (2k entries) and its threshold drops candidates
    by the same order; docs and total bits equal a sort by (order_key desc, doc asc)"""
    rng = np.random.default_rng(2)
    for trial in range(40):
        n = int(rng.integers(1, 400))
        totals = np.array(VALUES, np.float64)[rng.integers(0, len(VALUES), n)]
        docs = rng.permutation(1 << 20)[:n].astype(np.uint32)
        for k in (1, 2, 3, 7, 31, 32, 33, n):
            od, ot = oracle.topn_f64(totals, docs, k)
            ed, et = R.expected_topk(totals, docs, k)
            assert np.array_equal(od, ed), (trial, k)
            assert np.array_equal(R.bits(ot), R.bits(et)), (trial, k)   # the pushed values, NaN payloads included


def test_negative_zero_below_positive_zero():
    od, ot = oracle.topn_f64(np.array([-0.0, 0.0, -0.0, 0.0]), np.array([1, 9, 0, 8], np.uint32), 3)
    assert list(od) == [8, 9, 0] and list(R.bits(ot)) == [0, 0, 0x8000000000000000]


def test_nan_ranks_below_negative_infinity():
    od, _ = oracle.topn_f64(np.array([R.NAN_P, -np.inf, R.NAN_N, -R.F64_MAX]), np.array([0, 1, 2, 3], np.uint32), 4)
    assert list(od) == [3, 1, 0, 2]


def test_segment_merge_orders_by_total_cmp():
    """the Searcher / SignalSearcher merge (bm25.merge_fruits) keys totals like the device and the oracle: a +0.0 doc of
    segment 1 ranks above a -0.0 doc of segment 0, NaNs of either sign tie below -inf by (segment, doc), the offset is
    dropped after the merge"""
    from stract_b200.bm25 import merge_fruits
    p0 = (0, np.array([[4, 2, 7, 1]], np.uint32), np.array([[-0.0, R.NAN_P, -np.inf, 3.0]]), np.array([4], np.uint32))
    p1 = (1, np.array([[3, 0, 5, 9]], np.uint32), np.array([[0.0, R.NAN_N, 3.0, -R.SUB]]), np.array([4], np.uint32))
    segs, docs, tot = merge_fruits([p0, p1], 0, 8)
    assert list(zip(segs.tolist(), docs.tolist())) == [(0, 1), (1, 5), (1, 3), (0, 4), (1, 9), (0, 7), (0, 2), (1, 0)]
    assert list(R.bits(tot[:4])) == list(R.bits([3.0, 3.0, 0.0, -0.0]))
    segs, docs, _ = merge_fruits([p0, p1], 0, 3, offset=2)
    assert list(zip(segs.tolist(), docs.tolist())) == [(1, 3), (0, 4), (1, 9)]
