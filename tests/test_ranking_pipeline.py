"""The recall-stage mirror (stract_b200/ranking_pipeline.py) on the reference's own tests and hand cases; no GPU."""
import numpy as np

from stract_b200 import ranking_pipeline as RP
from stract_b200.bm25 import CORE_SIGNALS, NUMERIC_SIGNALS

U = RP.U32_MAX


def test_min_slop_reference():
    # term_distance.rs test_min_slop
    assert RP.min_slop([[13, 18, 22], [8, 15, 30], [9, 16]]) == 2


def test_min_slop_hand_cases():
    assert RP.min_slop([[3, 9]]) == U                      # one term: no pair
    assert RP.min_slop([]) == U
    assert RP.min_slop([[1, 5], []]) == U                  # an absent term (or one the document lacks)
    assert RP.min_slop([[7, 9], [2, 4]]) == U              # b only before a
    assert RP.min_slop([[4], [4]]) == U                    # equal positions never count
    assert RP.min_slop([[1, 4, 8], [1, 4, 8]]) == 3        # a duplicate term: its own next position
    assert RP.min_slop([[0, 10], [5, 11]]) == 1
    assert RP.min_slop([[0], [1], [9]]) == 8               # the max over the pairs
    assert RP.min_slop_two_positions([5, 6], [1, 2, 3, 7]) == 1


def test_min_slop_walk_equals_successor_search():
    """the two-cursor walk is the min over a of (smallest b > a) - a: the form the device kernel evaluates"""
    rng = np.random.default_rng(1)
    for _ in range(2000):
        a = sorted(set(rng.integers(0, 40, rng.integers(0, 8)).tolist()))
        b = sorted(set(rng.integers(0, 40, rng.integers(0, 8)).tolist()))
        succ = [min([y for y in b if y > x], default=None) for x in a]
        want = min([s - x for s, x in zip(succ, a) if s is not None], default=U)
        assert RP.min_slop_two_positions(a, b) == want, (a, b)


def test_score_slop():
    assert RP.score_slop(0) == 1.0 and RP.score_slop(3) == 0.25 and RP.score_slop(U) == 1.0 / 4294967296.0


def test_signal_enum_order():
    assert len(RP.SIGNAL_ENUM) == 46 and len(set(RP.SIGNAL_ENUM)) == 46
    assert RP.SIGNAL_ENUM[:3] == ["Bm25F", "Bm25Title", "TitleCoverage"]
    assert RP.SIGNAL_ENUM[24:26] == ["CrossEncoderSnippet", "CrossEncoderTitle"]
    assert RP.SIGNAL_ENUM[35:38] == ["QueryCentrality", "InboundSimilarity", "LambdaMart"]
    assert RP.SIGNAL_ENUM[-3:] == ["HasAds", "MinTitleSlop", "MinCleanBodySlop"]
    core = [n for n, *_ in CORE_SIGNALS] + [n for n, *_ in NUMERIC_SIGNALS]
    assert set(core) | set(RP.NON_CORE_COEFFICIENTS) == set(RP.SIGNAL_ENUM)
    # CoreSignalEnum keeps SignalEnum's relative order
    assert [n for n in RP.SIGNAL_ENUM if n in core] == [n for n, *_ in CORE_SIGNALS] + [n for n, *_ in NUMERIC_SIGNALS][:9] + \
        ["UrlDigits", "UrlSlashes", "LinkDensity", "HasAds"]


def test_default_coefficients():
    c = RP.default_coefficients()
    assert c["MinTitleSlop"] == 0.1 and c["MinCleanBodySlop"] == 0.1 and c["InboundSimilarity"] == 0.25
    assert c["HostCentrality"] == 2.0 and c["Bm25F"] == 0.1 and c["LambdaMart"] == 10.0


def test_pipeline_simple():
    """pipeline/mod.rs `simple`: 20 pages with HostCentrality { value: i, score: 1 / i } and that score as the initial one; the
    TitleDistance and BodyDistance stages keep the order 0, 1, ..., 19"""
    coefs = RP.default_coefficients()
    pages = []
    for i in range(20):
        s = 1.0 / i if i else float("inf")
        p = RP.Page(i, {"HostCentrality": (float(i), s)}, s, 1.0)
        p.min_slop = (U, U)
        pages.append(p)
    for field, name in ((0, "MinTitleSlop"), (1, "MinCleanBodySlop")):
        for p in pages:
            v = float(p.min_slop[field])
            p.signals[name] = (v, RP.score_slop(v))
        RP.update_scores(pages, coefs)
        RP.rank(pages)
    assert [p.key for p in pages] == list(range(20))


def test_update_scores_folds_in_signal_enum_order():
    """the fold runs in SignalEnum order, not in insertion order: 1e16 + 1 - 1e16 differs from 1e16 - 1e16 + 1"""
    coefs = {"Bm25F": 1.0, "Bm25Title": 1.0, "MinTitleSlop": 1.0}
    p = RP.Page(0, {"MinTitleSlop": (0.0, -1e16), "Bm25Title": (0.0, 1.0), "Bm25F": (0.0, 1e16)}, 0.0, 1.0)
    RP.update_scores([p], coefs)
    assert p.score == (1e16 + 1.0) + -1e16


def test_rank_is_stable_under_ties():
    pages = [RP.Page(k, {}, s, b) for k, s, b in [(0, 1.0, 2.0), (1, 2.0, 1.0), (2, 4.0, 1.0), (3, 0.5, 4.0), (4, 1.0, 1.0)]]
    RP.rank(pages)
    assert [p.key for p in pages] == [2, 0, 1, 3, 4]


def test_recall_stage_inbound_modifier():
    """InboundScorer adds InboundSimilarity (value = score), then the modifier multiplies the boost by value + 8 and re-ranks
    without re-summing"""
    coefs = RP.default_coefficients()
    pages = []
    for k in range(3):
        p = RP.Page(k, {"Bm25Title": (1.0, 1.0)}, 0.0063, 1.0)
        p.min_slop = (U, U)
        pages.append(p)
    inbound = {0: 0.0, 1: 2.0, 2: 1.0}
    out = RP.recall_stage(pages, coefs, inbound)
    assert [p.key for p in out] == [1, 2, 0]
    assert out[0].boost == 10.0 and out[2].boost == 8.0
    want = 0.0 + 1.0 * coefs["Bm25Title"]
    want = want + 2.0 * coefs["InboundSimilarity"]
    want = want + RP.score_slop(U) * 0.1
    want = want + RP.score_slop(U) * 0.1
    assert out[0].score == want
