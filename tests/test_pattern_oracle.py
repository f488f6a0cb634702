"""The pattern / optic oracle (tests/pattern_oracle.py) pinned on the reference: the intersection_with_slop KATs of
core/src/query/pattern_query/scorer.rs:423-438, the quirks of NormalPatternScorer and pattern_scorer's branches, and the
rule / filter composition of core/src/query/optic.rs.  No GPU, no library.

The end-to-end optic tests of optic.rs (special_pattern_syntax, wildcard_edge_cases, empty_double_anchor, pattern_same_phrase,
site_double_anchor, discard_double_matching, test_site_in_domain_rule, discard_all_discard_like) index whole web pages through
Stract's stemming, language-detecting tokenizers and its site / domain normalisation; their token streams are not derived
here, so those scenarios are unpinned.  The quirks they exercise are pinned below on hand-made token streams."""
import pattern_oracle as PO

MAX = PO.U32_MAX


def test_intersection_with_slop_kats():
    kats = [([20, 75, 77], [18, 21, 60], [21, 60], MAX), ([21, 60], [50, 61], [61], 1), ([1, 2, 3], [], [], 1),
            ([], [1, 2, 3], [], 1), ([1, 2, 3], [4, 5, 6], [4], 1), ([1, 2, 3], [4, 5, 6], [4, 5, 6], MAX),
            ([20, 75, 77], [18, 21, 60], [21, 60], MAX), ([21, 60], [61, 62], [61, 62], 2), ([60], [61, 62], [61, 62], 2)]
    for left, right, want, slop in kats:
        assert PO.intersection_with_slop(left, right, slop) == want
        # the order-free set form the kernel evaluates lane by lane
        assert [r for r in right if any(max(r - slop, 0) <= l <= r for l in left)] == want


def test_set_form_equals_the_walk_on_random_lists():
    import random
    rnd = random.Random(3)
    for _ in range(3000):
        left = sorted(rnd.sample(range(60), rnd.randint(0, 12)))
        right = sorted(rnd.sample(range(60), rnd.randint(0, 12)))
        slop = rnd.choice([0, 1, 2, 5, MAX])
        want = [r for r in right if any(max(r - slop, 0) <= l <= r for l in left)]
        assert PO.intersection_with_slop(left, right, slop) == want


A, B, C, X = 1, 2, 3, 9


def docs_of(field, parts, terms, counts=None):
    counts = [len(t) for t in field] if counts is None else counts
    return PO.pattern_docs(field, list(parts), terms, counts)


def test_branches():
    field = [[A, B], [], [B], [C, C, C]]
    assert docs_of(field, "", []) == []                                  # empty pattern
    assert docs_of(field, "*", []) == [0, 1, 2, 3]                       # AllScorer
    assert docs_of(field, "|*|", []) == [0, 1, 2, 3]                     # "|*|": a wildcard, no terms
    assert docs_of(field, "||", []) == [1]                               # EmptyFieldScorer
    assert docs_of(field, "|", [], counts=[2, None, 1, 3]) == [1]         # a missing count is 0
    assert docs_of(field, "T", [None]) == []                             # a term the segment lacks
    assert docs_of(field, "TT", [A, None]) == []
    assert docs_of(field, "T", [C]) == [3]                               # the single-term shortcut


def test_normal_scorer_quirks():
    f = [[A, X, A, B], [A, A], [X, A], [B, A], [A, X, X, B], [A, B, X]]
    assert docs_of(f, "|TT", [A, B]) == [0, 5]       # the start anchor checks term 0's FIRST position, not the chain's start
    assert docs_of(f, "TT", [A, A]) == [0, 1, 2, 3, 4, 5]   # distance 0 is accepted: "a a" matches one a
    assert docs_of(f, "*T", [B]) == docs_of(f, "T", [B]) == [0, 3, 4, 5]   # a leading wildcard does nothing
    assert docs_of(f, "T*T", [A, B]) == [0, 4, 5]    # wildcard: any distance, still ordered
    assert docs_of(f, "TT", [B, A]) == [3]
    assert docs_of(f, "TT|", [A, B]) == [0]          # end anchor: the last position of the last term is num_tokens - 1
    assert docs_of(f, "T|T", [A, B]) == [0, 5]       # a middle anchor is ignored
    # the end anchor reads the last term's RAW list, not the chain: "a b|" matches when b's last position is the end
    g = [[A, B, X, B], [A, X, B]]
    assert docs_of(g, "TT|", [A, B]) == [0]
    # the count column decides, not the list: a count that disagrees with the tokens
    assert docs_of(g, "T|", [B], counts=[5, 3]) == [1]
    # num_tokens 0 wraps: (0 - 1) as u32 = u32::MAX, which no position equals
    assert docs_of([[A]], "T|", [A], counts=[0]) == []


def test_rule_composition_and_boosts():
    sets = {"a": {1, 2, 3}, "b": {2, 3, 4}, "c": {9}}
    m = lambda name: sets[name]
    assert PO.rule_docs([["a", "b"], ["c"]], m) == {2, 3, 9}          # OR over blocks of the AND within a block
    assert PO.rule_docs([[], ["c"]], m) == {9}                         # empty blocks are dropped
    assert PO.rule_docs([[]], m) is None                               # no block: no rule
    # SignalComputer::boosts: downrank > boost -> 1 / (1 + diff), else boost - downrank + 1
    assert PO.boost_factor(2, [({2}, 3.0), ({2}, -1.0)]) == 3.0
    assert PO.boost_factor(2, [({2}, 1.0), ({2}, -4.0)]) == 1.0 / (1.0 + 3.0)
    assert PO.boost_factor(5, [({2}, 1.0)]) == 1.0
    got = PO.optic_topk([(1, 2.0), (2, 2.0), (3, 1.0), (4, 0.5)], 3, [({3}, 3.0)], exclude={1}, require={2, 3, 4})
    assert got == [(4.0, 3), (2.0, 2), (0.5, 4)]
