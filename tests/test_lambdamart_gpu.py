"""sb200_lambdamart_* (lambdamart.cu) against tests/lambdamart_oracle.py: every output bit (any NaN equal to any NaN), every load
error, bad arguments, and the recall stage's LambdaMART step in stract_b200/ranking_pipeline.py.  The check_* functions also
run, reduced, on the CPU SIMT emulator (test_lambdamart_emulated.py)."""
import ctypes as C
import os

import numpy as np
import pytest

import lambdamart_oracle as O
from stract_b200 import _lib
from stract_b200 import ranking_pipeline as RP
from stract_b200._lib import Sb200Error
from stract_b200.lambdamart import LambdaMART

pytestmark = pytest.mark.gpu
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lambdamart.txt")
EFORMAT, EINVAL = -6, -1


def same(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    nan = np.isnan(got) & np.isnan(want)
    return got.shape == want.shape and bool(np.all(nan | (got.view(np.uint64) == want.view(np.uint64))))


def check_model(text, X, max_depth=None):
    """the library's predict equals the oracle's vectorised walk bit for bit; counts match the oracle's model"""
    model, om = LambdaMART.parse(text), O.Model(text)
    want, _ = O.predict_numpy(om, X)
    got = model.predict(X)
    bad = np.flatnonzero(~(np.isnan(got) & np.isnan(want)) & (got.view(np.uint64) != want.view(np.uint64)))
    assert bad.size == 0, (bad[:5], got[bad[:5]], want[bad[:5]])
    assert model.n_trees == len(om.trees) and model.features == [O.SIGNAL_ENUM[f] for f in om.features]
    assert model.info["n_leaves"] == om.n_slots()
    if max_depth is not None:
        assert model.info["max_depth"] == max_depth
    assert model.last_stats["docs"] == len(X)
    return model, got


def check_fixture(n_rows=2_000, seed=1):
    model = LambdaMART.open(FIXTURE)
    assert model.n_trees == 50 and len(model.features) == 29
    p = model.predict(np.array([O.simple_row()]))[0]
    assert int(p * 1000) == 1050 and int(np.float64(p).view(np.uint64)) == O.SIMPLE_BITS
    om = O.Model(open(FIXTURE).read())
    th = sorted({n.threshold for t in om.trees for n in t.nodes})
    check_model(open(FIXTURE).read(), O.random_rows(np.random.default_rng(seed), n_rows, th))


def check_synthetic(cases):
    """cases: (seed, n_trees, leaves, chain_every, n_docs); also a header with repeated features"""
    for seed, n_trees, leaves, chain_every, n_docs in cases:
        rng = np.random.default_rng(seed)
        text, th = O.random_model(rng, n_trees, leaves, chain_every=chain_every)
        check_model(text, O.random_rows(rng, n_docs, th))
    rng = np.random.default_rng(99)
    names = ["bm25_title", "bm25_clean_body", "bm25_title", "host_centrality", "bm25_clean_body"]
    text, th = O.random_model(rng, 40, (2, 31), feature_names=names)
    check_model(text, O.random_rows(rng, 300, th))


def check_chain(n_leaves, n_docs):
    rng = np.random.default_rng(n_leaves)
    text, th = O.random_model(rng, 3, n_leaves, chain_every=1)
    check_model(text, O.random_rows(rng, n_docs, th), max_depth=n_leaves - 1)


def check_batch_sizes(sizes):
    text = open(FIXTURE).read()
    om = O.Model(text)
    th = sorted({n.threshold for t in om.trees for n in t.nodes})
    model = LambdaMART.parse(text)
    rng = np.random.default_rng(5)
    for n in sizes:
        X = O.random_rows(rng, n, th)
        assert same(model.predict(X), O.predict_numpy(om, X)[0]), n


def load_error_cases():
    """(model text or bytes, what the reference does): each has exactly one defect"""
    stump = ["split_feature=1", "threshold=2.5", "left_child=-1", "right_child=-2", "leaf_value=-0.5 0.25"]

    def hand(*trees, header="feature_names=bm25_title bm25_clean_body", sep="\n\n", tail="\n\nend of trees\n"):
        return "tree\n" + header + "\n\n" + sep.join("\n".join(t) for t in trees) + tail

    def edit(**kv):
        return [f"{k}={kv[k]}" if k in kv else x for x in stump for k in [x.split("=")[0]]]
    return [
        (hand(stump, header="objective=lambdarank"), "NoFeatures"),
        (hand(stump, header="feature_names=bm25_title bm25"), "UnknownSignal"),
        (hand(stump, tail="\n\n"), "NoEndOfTrees"),
        (hand(stump).encode() + b"\xc3", "Io"),
        (hand(edit(threshold=" 2.5")), "ParseFloat"),
        (hand(edit(leaf_value="1_0 2")), "ParseFloat"),
        (hand(edit(split_feature="-1")), "ParseInt"),
        (hand(edit(right_child="2147483648")), "ParseInt"),
        ("tree\nfeature_names=bm25_title\nend of trees\n", "panic"),            # no empty line after the header
        (hand(edit(split_feature="2")), "panic"),                                # beyond the header
        (hand(edit(threshold="1 2 3")), "panic"),                                # more thresholds than node slots
        (hand(stump, stump, sep="\n\n\n\n"), "panic"),                           # an empty tree
        (hand([x for x in stump if not x.startswith("split_feature")]), "panic"),   # the root has no feature
        (hand([x for x in stump if not x.startswith("right_child")]), "panic"),     # a missing child
        (hand(edit(left_child="5")), "panic"),                                   # a node index out of range
        (hand(edit(left_child="-9")), "panic"),                                  # a leaf index out of range
        (hand(edit(left_child="0")), "loops forever"),                           # a cycle
    ]


def oracle_outcome(text):
    try:
        m = O.Model(text)
    except O.LambdaError as e:
        return e.kind
    e = m.reachable_failure()
    return e.kind if e is not None else None


def check_load_errors():
    for text, kind in load_error_cases():
        assert oracle_outcome(text) == kind, (text, kind)
        with pytest.raises(Sb200Error) as ei:
            LambdaMART.parse(text)
        assert ei.value.code == EFORMAT and str(ei.value).split(": ", 1)[1].startswith(kind), (kind, str(ei.value))
    # malformed nodes no path reaches are accepted; a NaN threshold never goes left
    for text in ["tree\nfeature_names=bm25_clean_body\n\nsplit_feature=0\nthreshold=nan\nright_child=-2\nleaf_value=1 2\n\nend of trees\n",
                 "tree\nfeature_names=bm25_clean_body\n\nsplit_feature=0\nthreshold=1\nleft_child=-1 9\nright_child=-2\nleaf_value=1 2\n\n"
                 "end of trees\n"]:
        assert oracle_outcome(text) is None
        check_model(text, O.random_rows(np.random.default_rng(0), 50, [1.0]))
    # zero trees: 0.0 / 0.0
    z = LambdaMART.parse("tree\nfeature_names=bm25_title\n\nend of trees\n")
    assert z.n_trees == 0 and np.isnan(z.predict(np.zeros((3, 46)))).all()


def check_bad_args():
    L = _lib.lib()
    h = C.c_void_p()
    assert L.sb200_lambdamart_load(b"x", 1, None) == EINVAL
    assert L.sb200_lambdamart_load(None, 5, C.byref(h)) == EINVAL
    assert L.sb200_lambdamart_predict(None, None, 0, None, None) == EINVAL
    assert L.sb200_lambdamart_get_info(None, None) == EINVAL
    model = LambdaMART.open(FIXTURE)
    out = np.zeros(4)
    assert L.sb200_lambdamart_predict(model._h, None, 4, out.ctypes.data, None) == EINVAL
    assert L.sb200_lambdamart_predict(model._h, np.zeros((4, 46)).ctypes.data, 4, None, None) == EINVAL
    assert L.sb200_lambdamart_features(model._h, None, 3) == EINVAL
    assert L.sb200_lambdamart_predict(model._h, None, 0, None, None) == 0
    with pytest.raises(ValueError):
        model.predict(np.zeros((4, 45)))


def check_device_inputs(n=5_000):
    import torch
    text = open(FIXTURE).read()
    om = O.Model(text)
    th = sorted({n.threshold for t in om.trees for n in t.nodes})
    X = O.random_rows(np.random.default_rng(8), n, th)
    model = LambdaMART.parse(text)
    got = model.predict(torch.from_numpy(X).cuda())
    assert got.is_cuda and same(got.cpu().numpy(), model.predict(X)) and same(model.predict(X), O.predict_numpy(om, X)[0])


def oracle_stage(pages, coefficients, om, offset):
    """the LambdaMART stage restated over the oracle's predictions"""
    if offset > RP.LAMBDAMART_TOP:
        return pages
    top = pages[:RP.LAMBDAMART_TOP]
    for p in top:
        row = [0.0] * len(O.SIGNAL_ENUM)
        for name, (_v, s) in p.signals.items():
            row[O.SIGNAL_ENUM.index(name)] = s
        v = om.predict(row)
        p.signals["LambdaMart"] = (v, v)
    RP.update_scores(top, coefficients)
    RP.rank(top)
    return top + pages[len(top):]


def check_pipeline(n_docs=4_000, nq=12, k=40, seed=5, long_doc=600):
    import copy
    import test_recall_webpages_gpu as W
    fields, comp, cols, rng = W.build(seed, n_docs, long_doc)
    sf, st, sb = W.random_slots(rng, nq)
    td, tt, tn = comp.top_docs_batch(sf, st, k, slot_boost=sb)
    wp = comp.ranking_webpages(sf, st, td, tn, slot_boost=sb)
    coefs = RP.default_coefficients()
    inbound = {d: float(x) for d, x in enumerate(rng.random(n_docs))}
    model, om = LambdaMART.open(FIXTURE), O.Model(open(FIXTURE).read())
    per_query = [RP.pages_from_webpages(wp, q, td[q], int(tn[q]), tt[q]) for q in range(nq)]
    assert max(len(p) for p in per_query) > RP.LAMBDAMART_TOP
    key = lambda ps: [(p.key, float(p.score), float(p.boost)) for p in ps]   # noqa: E731
    batch = RP.recall_stage_batch(copy.deepcopy(per_query), coefs, inbound, model, 0)
    for q in range(nq):
        plain = RP.recall_stage(copy.deepcopy(per_query[q]), coefs, inbound)
        got = RP.recall_stage(copy.deepcopy(per_query[q]), coefs, inbound, lambdamart=model)
        want = oracle_stage(RP.recall_stage(copy.deepcopy(per_query[q]), coefs, inbound), coefs, om, 0)
        assert [p.key for p in got] == [p.key for p in want], q
        assert all(same(a.score, b.score) and same(a.boost, b.boost) for a, b in zip(got, want)), q
        assert all(same(a.signals["LambdaMart"][0], b.signals["LambdaMart"][0]) for a, b in zip(got[:20], want[:20]))
        top = RP.LAMBDAMART_TOP
        assert key(got[top:]) == key(plain[top:]) and {p.key for p in got[:top]} == {p.key for p in plain[:top]}, q
        skipped = RP.recall_stage(copy.deepcopy(per_query[q]), coefs, inbound, lambdamart=model, offset=21)
        assert key(skipped) == key(plain) and all("LambdaMart" not in p.signals for p in skipped), q
        at20 = RP.recall_stage(copy.deepcopy(per_query[q]), coefs, inbound, lambdamart=model, offset=20)
        assert key(at20) == key(got), q
        assert key(batch[q]) == key(got), q


def test_lambdamart_fixture():
    check_fixture()


def test_lambdamart_synthetic():
    check_synthetic([(1, 1, 2, 0, 500), (2, 10, (2, 8), 0, 2_000), (3, 300, (2, 63), 7, 3_000), (4, 2_000, (2, 255), 50, 1_500),
                     (5, 120, 255, 0, 2_000)])


def test_lambdamart_chains():
    check_chain(300, 1_000)
    check_chain(700, 500)


def test_lambdamart_global_tree():
    # ~20 000 leaves: 480 KB of records and leaves, far above the 32 KB shared tree buffer, walked from global memory
    rng = np.random.default_rng(12)
    text, th = O.random_model(rng, 3, (19_000, 20_500))
    check_model(text, O.random_rows(rng, 3_000, th))


def test_lambdamart_batch_sizes():
    check_batch_sizes([1, 31, 32, 33, 127, 128, 129, 100_003])


def test_lambdamart_device_inputs():
    check_device_inputs()


def test_lambdamart_load_errors():
    check_load_errors()


def test_lambdamart_bad_args():
    check_bad_args()


def test_lambdamart_recall_stage():
    check_pipeline()
