"""The LambdaMART restatement (tests/lambdamart_oracle.py) pinned on the reference's `simple` test and on the parser's quirks."""
import math
import struct

import pytest

import lambdamart_oracle as O

FIXTURE = __file__.rsplit("/", 1)[0] + "/golden/lambdamart.txt"


def bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def hand(*trees, header="feature_names=bm25_title bm25_clean_body", sep="\n\n", tail="\n\nend of trees\n"):
    """a model text from tree bodies (lists of lines)"""
    return "tree\n" + header + "\n\n" + sep.join("\n".join(t) for t in trees) + tail


STUMP = ["Tree=0", "split_feature=1", "threshold=2.5", "left_child=-1", "right_child=-2", "leaf_value=-0.5 0.25"]


def row(title=0.0, body=0.0):
    r = [0.0] * len(O.SIGNAL_ENUM)
    r[O.SIGNAL_ENUM.index("Bm25Title")] = title
    r[O.SIGNAL_ENUM.index("Bm25CleanBody")] = body
    return r


def test_simple_pinned():
    m = O.Model(open(FIXTURE, "rb").read())
    p = m.predict(O.simple_row())
    assert int(p * 1000) == 1050
    assert bits(p) == O.SIMPLE_BITS and p == 1.0505828267036237


def test_fixture_shape():
    m = O.Model(open(FIXTURE).read())
    assert len(m.trees) == 50 and len(m.features) == 29 and len(set(m.features)) == 29
    assert m.reachable_failure() is None


def test_stump_offset_and_edge():
    m = O.Model(hand(STUMP))
    off = abs(-0.5) + 1.0
    assert m.predict(row(body=2.5)) == -0.5 + off          # value <= threshold goes left
    assert m.predict(row(body=2.6)) == 0.25 + off
    assert m.predict(row(body=math.nan)) == 0.25 + off     # NaN goes right


def test_one_or_two_blank_lines_between_trees():
    two = O.Model(hand(STUMP, STUMP, sep="\n\n\n"))
    one = O.Model(hand(STUMP, STUMP, sep="\n\n"))
    assert len(two.trees) == 2 and len(one.trees) == 2      # end_tree + 2 skips the blank line or the Tree= line
    assert two.predict(row(body=3.0)) == one.predict(row(body=3.0))


def test_three_blank_lines_make_an_empty_tree_that_panics():
    m = O.Model(hand(STUMP, STUMP, sep="\n\n\n\n"))
    assert len(m.trees) == 3 and m.trees[1].nodes == []
    assert isinstance(m.reachable_failure(), O.Panic)
    with pytest.raises(O.Panic):
        m.predict(row())


def test_repeated_keys_append():
    split = ["Tree=0", "split_feature=1", "threshold=2.5", "left_child=-1", "right_child=-2", "leaf_value=-0.5", "leaf_value=0.25"]
    hdr = "feature_names=bm25_title\nfeature_names=bm25_clean_body"
    a, b = O.Model(hand(split, header=hdr)), O.Model(hand(STUMP))
    assert a.features == b.features and a.predict(row(body=9.0)) == b.predict(row(body=9.0))


def test_short_threshold_list_keeps_zero():
    t = ["split_feature=1 0", "threshold=5.0", "left_child=1 -2", "right_child=-1 -3", "leaf_value=1.0 2.0 3.0"]
    m = O.Model(hand(t))
    assert m.trees[0].nodes[1].threshold == 0.0
    # body 1.0 <= 5 -> node 1; title 0.0 <= 0.0 -> leaf 1; title 0.1 -> leaf 2
    assert m.predict(row(title=0.0, body=1.0)) == 2.0 + 2.0 and m.predict(row(title=0.1, body=1.0)) == 3.0 + 2.0


@pytest.mark.parametrize("leaves,offset", [("-0.5 0.25", 1.5), ("0.5 0.25", 1.25), ("nan 0.25", 1.25), ("0.25 nan", math.nan)])
def test_offset_fold(leaves, offset):
    t = STUMP[:-1] + ["leaf_value=" + leaves]
    m = O.Model(hand(t))
    lv = [O.parse_f64(x) for x in leaves.split(" ")]
    got = [n.leaf_value for n in m.trees[0].nodes]
    for g, v in zip(got, lv):
        assert (math.isnan(g) and (math.isnan(v) or math.isnan(offset))) or g == v + offset


def test_crlf():
    a = O.Model(hand(STUMP).replace("\n", "\r\n"))
    assert a.predict(row(body=3.0)) == O.Model(hand(STUMP)).predict(row(body=3.0))


@pytest.mark.parametrize("tok", [" 1", "1 ", "1_0", "0x1p3", "nan(1)", "1e", ".", "e5", "1.5.", "--1", ""])
def test_rust_rejected_floats(tok):
    with pytest.raises(O.ParseFloat):
        O.Model(hand(STUMP[:2] + ["threshold=" + tok] + STUMP[3:]))


@pytest.mark.parametrize("tok,value", [("inf", math.inf), ("-Infinity", -math.inf), ("NaN", math.nan), ("+1", 1.0), ("1.", 1.0),
                                       (".5", 0.5), ("1E+2", 100.0)])
def test_rust_accepted_floats(tok, value):
    m = O.Model(hand(STUMP[:2] + ["threshold=" + tok] + STUMP[3:]))
    t = m.trees[0].nodes[0].threshold
    assert (math.isnan(t) and math.isnan(value)) or t == value


@pytest.mark.parametrize("line", ["split_feature=-1", "split_feature= 1", "left_child=1.0", "right_child=2147483648", "left_child=+"])
def test_rust_rejected_ints(line):
    key = line.split("=")[0]
    body = [x for x in STUMP if not x.startswith(key + "=")] + [line]
    with pytest.raises(O.ParseInt):
        O.Model(hand(body))


def test_reference_errors():
    with pytest.raises(O.NoFeatures):
        O.Model(hand(STUMP, header="objective=lambdarank"))
    with pytest.raises(O.UnknownSignal):
        O.Model(hand(STUMP, header="feature_names=bm25_title Bm25CleanBody"))
    with pytest.raises(O.NoEndOfTrees):
        O.Model(hand(STUMP, tail="\n\n"))
    with pytest.raises(O.Io):
        O.Model(hand(STUMP).encode() + b"\xff")
    with pytest.raises(O.Panic):                       # no empty line after the header
        O.Model("tree\nfeature_names=bm25_title")
    with pytest.raises(O.Panic):                       # split_feature beyond the header
        O.Model(hand(["split_feature=2"] + STUMP[2:]))
    with pytest.raises(O.Panic):                       # more split features than node slots
        O.Model(hand(["split_feature=1 1 1"] + STUMP[2:]))


def test_walk_failures():
    no_feature = ["threshold=1.0", "left_child=-1", "right_child=-2", "leaf_value=1 2"]
    assert isinstance(O.Model(hand(no_feature)).reachable_failure(), O.Panic)
    cycle = ["split_feature=1 0", "threshold=1.0 2.0", "left_child=1 -1", "right_child=-2 0", "leaf_value=1 2"]
    m = O.Model(hand(cycle))
    assert isinstance(m.reachable_failure(), O.Loop)
    with pytest.raises(O.Loop):
        m.predict(row(title=5.0, body=0.5))            # node 0 left -> node 1 right -> node 0 ...
    assert m.predict(row(title=0.0, body=0.5)) == 1.0 + 2.0   # the walks that leave the cycle still end
    nan_left = ["split_feature=1", "threshold=nan", "right_child=-2", "leaf_value=1 2"]
    assert O.Model(hand(nan_left)).reachable_failure() is None   # a NaN threshold never goes left
    unreachable = ["split_feature=1", "threshold=1.0", "left_child=-1 7", "right_child=-2", "leaf_value=1 2"]
    assert O.Model(hand(unreachable)).reachable_failure() is None


def test_zero_trees_predict_nan():
    m = O.Model("tree\nfeature_names=bm25_title\n\nend of trees\n")
    assert m.trees == [] and math.isnan(m.predict(row()))


def test_trim_and_lines():
    assert O.rust_lines("a\r\nb\r\r\n\nc\r") == ["a", "b\r", "", "c\r"]
    assert O.rust_trim("　 end of trees\t\x85") == "end of trees" and O.rust_trim("\x1cend of trees") != "end of trees"
