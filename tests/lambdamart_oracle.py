"""A plain restatement of Stract's LambdaMART (core/src/ranking/models/lambdamart.rs): the reference's structs (Node with tagged
Node / Leaf children in one slot array per tree), its parser and its walk.  It does not use the library.  It raises the reference's
error kinds, and Panic / Loop where the reference would panic or loop forever.  Test infrastructure only."""
import math
import re

SIGNAL_ENUM = ["Bm25F", "Bm25Title", "TitleCoverage", "Bm25TitleBigrams", "Bm25TitleTrigrams", "Bm25CleanBody", "CleanBodyCoverage",
               "Bm25CleanBodyBigrams", "Bm25CleanBodyTrigrams", "Bm25StemmedTitle", "Bm25StemmedCleanBody", "Bm25AllBody", "Bm25Keywords",
               "Bm25BacklinkText", "IdfSumUrl", "IdfSumSite", "IdfSumDomain", "IdfSumSiteNoTokenizer", "IdfSumDomainNoTokenizer",
               "IdfSumDomainNameNoTokenizer", "IdfSumDomainIfHomepage", "IdfSumDomainNameIfHomepageNoTokenizer",
               "IdfSumDomainIfHomepageNoTokenizer", "IdfSumTitleIfHomepage", "CrossEncoderSnippet", "CrossEncoderTitle", "HostCentrality",
               "HostCentralityRank", "PageCentrality", "PageCentralityRank", "IsHomepage", "FetchTimeMs", "UpdateTimestamp",
               "TrackerScore", "Region", "QueryCentrality", "InboundSimilarity", "LambdaMart", "UrlDigits", "UrlSlashes", "LinkDensity",
               "TitleEmbeddingSimilarity", "KeywordEmbeddingSimilarity", "HasAds", "MinTitleSlop", "MinCleanBodySlop"]


def snake_case(name):
    """serde's rename_all = "snake_case": '_' before every uppercase letter but the first, then lowercase"""
    return "".join(("_" if i and c.isupper() else "") + c.lower() for i, c in enumerate(name))


FROM_STR = {snake_case(n): i for i, n in enumerate(SIGNAL_ENUM)}


class LambdaError(Exception):
    kind = None


class NoFeatures(LambdaError):
    kind = "NoFeatures"


class NoEndOfTrees(LambdaError):
    kind = "NoEndOfTrees"


class ParseInt(LambdaError):
    kind = "ParseInt"


class ParseFloat(LambdaError):
    kind = "ParseFloat"


class UnknownSignal(LambdaError):
    kind = "UnknownSignal"


class Io(LambdaError):
    kind = "Io"


class Panic(LambdaError):
    """the reference panics (an unwrap on None / Err, an index out of bounds)"""
    kind = "panic"


class Loop(LambdaError):
    """the reference walks a cycle forever"""
    kind = "loops forever"


def rust_lines(s):
    """str::lines: split on '\n', one '\r' before it dropped, no empty line after a final '\n'"""
    parts = s.split("\n")
    last = parts.pop()
    out = [p[:-1] if p.endswith("\r") else p for p in parts]
    if last:
        out.append(last)
    return out


# char::is_whitespace
_WS = {chr(c) for c in [*range(0x09, 0x0E), 0x20, 0x85, 0xA0, 0x1680, *range(0x2000, 0x200B), 0x2028, 0x2029, 0x202F, 0x205F, 0x3000]}


def rust_trim(s):
    """str::trim: char::is_whitespace at both ends"""
    a, b = 0, len(s)
    while a < b and s[a] in _WS:
        a += 1
    while b > a and s[b - 1] in _WS:
        b -= 1
    return s[a:b]


def parse_usize(tok):
    if not re.fullmatch(r"\+?[0-9]+", tok):
        raise ParseInt(tok)
    v = int(tok)
    if v >= 1 << 64:
        raise ParseInt(tok)
    return v


def parse_i32(tok):
    if not re.fullmatch(r"[+-]?[0-9]+", tok):
        raise ParseInt(tok)
    v = int(tok)
    if not -(1 << 31) <= v < 1 << 31:
        raise ParseInt(tok)
    return v


def parse_f64(tok):
    """<f64 as FromStr>"""
    m = re.fullmatch(r"([+-]?)(inf|infinity|nan)", tok, re.I)
    if m:
        v = math.inf if m.group(2).lower() != "nan" else math.nan
        return -v if m.group(1) == "-" else v
    if not re.fullmatch(r"[+-]?([0-9]+\.?[0-9]*|\.[0-9]+)([eE][+-]?[0-9]+)?", tok):
        raise ParseFloat(tok)
    return float(tok)


class Node:
    """NodeOrLeaf children: ("node", i) / ("leaf", i) or None"""

    def __init__(self, leaf_value):
        self.threshold = 0.0
        self.feature = None
        self.leaf_value = leaf_value
        self.left = None
        self.right = None


def _child(tok):
    c = parse_i32(tok)
    return ("leaf", -c - 1) if c < 0 else ("node", c)


def _set(nodes, values, attr):
    for i, v in enumerate(values):
        if i >= len(nodes):
            raise Panic(f"index out of bounds: {attr} {i} for {len(nodes)} nodes")
        setattr(nodes[i], attr, v)


class Tree:
    def __init__(self, s, header):
        feats, thr, leaves, lefts, rights = [], [], [], [], []
        for line in rust_lines(s):
            if "=" not in line:
                continue
            key, value = line.split("=", 1)
            toks = value.split(" ")
            if key == "split_feature":
                for t in toks:
                    i = parse_usize(t)
                    if i >= len(header):
                        raise Panic(f"index out of bounds: split_feature {i}")
                    feats.append(header[i])
            elif key == "threshold":
                thr += [parse_f64(t) for t in toks]
            elif key == "leaf_value":
                leaves += [parse_f64(t) for t in toks]
            elif key == "left_child":
                lefts += [_child(t) for t in toks]
            elif key == "right_child":
                rights += [_child(t) for t in toks]
        offset = None
        for v in leaves:
            offset = v if offset is None else (offset if offset < v else v)
        if offset is not None:
            offset = abs(offset) + 1.0
        self.nodes = [Node(v + offset) for v in leaves]
        _set(self.nodes, feats, "feature")
        _set(self.nodes, thr, "threshold")
        _set(self.nodes, lefts, "left")
        _set(self.nodes, rights, "right")

    def _at(self, i):
        if i >= len(self.nodes):
            raise Panic(f"index out of bounds: node {i} of {len(self.nodes)}")
        return self.nodes[i]

    def predict(self, features):
        """Tree::predict(...).unwrap(); `features` is indexable by SignalEnum ordinal.  A walk longer than the slot count is a cycle."""
        node = self._at(0)
        for _ in range(len(self.nodes) + 1):
            if node.feature is None:
                raise Panic("LeafNotFound")
            nxt = node.left if features[node.feature] <= node.threshold else node.right
            if nxt is None:
                raise Panic("LeafNotFound")
            kind, i = nxt
            if kind == "leaf":
                return self._at(i).leaf_value
            node = self._at(i)
        raise Loop("cycle")

    def reachable_failure(self):
        """the error the walk meets on some path from the root, or None: what the library refuses at load.  A left edge exists
        unless the threshold is NaN; the right edge always exists (a NaN value goes right)."""
        try:
            state = {}

            def go(i):
                node = self._at(i)
                if state.get(i) == 1:
                    raise Loop("cycle")
                if state.get(i) == 2:
                    return
                state[i] = 1
                if node.feature is None:
                    raise Panic("LeafNotFound")
                for c in ([] if math.isnan(node.threshold) else [node.left]) + [node.right]:
                    if c is None:
                        raise Panic("LeafNotFound")
                    if c[0] == "leaf":
                        self._at(c[1])
                    else:
                        go(c[1])
                state[i] = 2
            go(0)
        except (Panic, Loop) as e:
            return e
        return None


class Model:
    """LambdaMART::parse"""

    def __init__(self, text):
        if isinstance(text, bytes):
            try:
                text = text.decode("utf-8")
            except UnicodeDecodeError:
                raise Io("stream did not contain valid UTF-8")
        lines = rust_lines(text)
        end_header = next((i for i, x in enumerate(lines) if x == ""), None)
        if end_header is None:
            raise Panic("no empty line after the header")
        self.features = []
        for lin in rust_lines("\n".join(lines[:end_header])):
            if "=" in lin:
                key, value = lin.split("=", 1)
                if key == "feature_names":
                    for name in value.split(" "):
                        if name not in FROM_STR:
                            raise UnknownSignal(name)
                        self.features.append(FROM_STR[name])
        if not self.features:
            raise NoFeatures()
        end_trees = next((i for i, x in enumerate(lines) if rust_trim(x) == "end of trees"), None)
        if end_trees is None:
            raise NoEndOfTrees()
        self.trees = []
        start = end_header + 1
        while start < end_trees:
            end = next((i for i in range(start, len(lines)) if lines[i] == ""), None)
            if end is None:
                raise Panic("no empty line after a tree")
            self.trees.append(Tree("\n".join(lines[start:end]), self.features))
            start = end + 2

    def reachable_failure(self):
        for t in self.trees:
            e = t.reachable_failure()
            if e is not None:
                return e
        return None

    def predict(self, features):
        """LambdaMART::predict: sum of the trees in order (from 0.0) divided by the number of trees"""
        acc = 0.0
        for t in self.trees:
            acc += t.predict(features)
        return acc / len(self.trees) if self.trees else math.nan

    def n_slots(self):
        return sum(len(t.nodes) for t in self.trees)


def same_bits(a, b):
    """bit equality, any NaN equal to any NaN (the NaN payload a sum produces is the hardware's)"""
    import struct
    if math.isnan(a) and math.isnan(b):
        return True
    return struct.pack("<d", a) == struct.pack("<d", b)


def predict_numpy(model, X):
    """LambdaMART::predict over every row of X [n][46] at once, for models without reachable failures: per tree a vectorised
    walk, the trees added to one f64 vector in tree order (the same sequential sum).  Also returns the node visits."""
    import numpy as np
    X = np.asarray(X, np.float64)
    n = X.shape[0]
    acc = np.zeros(n)
    rows = np.arange(n)
    visits = 0
    for t in model.trees:
        m = len(t.nodes)
        feat = np.array([nd.feature if nd.feature is not None else 0 for nd in t.nodes], np.int64)
        thr = np.array([nd.threshold for nd in t.nodes])
        leafv = np.array([nd.leaf_value for nd in t.nodes])

        def enc(c):
            return -1 - c[1] if c is not None and c[0] == "leaf" else (c[1] if c is not None else 0)
        left = np.array([enc(nd.left) for nd in t.nodes], np.int64)
        right = np.array([enc(nd.right) for nd in t.nodes], np.int64)
        cur = np.zeros(n, np.int64)
        out = np.zeros(n)
        live = rows
        steps = 0
        while live.size:
            c = cur[live]
            visits += live.size
            nxt = np.where(X[live, feat[c]] <= thr[c], left[c], right[c])
            done = nxt < 0
            out[live[done]] = leafv[-1 - nxt[done]]
            cur[live[~done]] = nxt[~done]
            live = live[~done]
            steps += 1
            assert steps <= m + 1, "cycle"
        acc = acc + out
    return (acc / len(model.trees) if model.trees else np.full(n, np.nan)), visits


def lightgbm_tree(rng, n_leaves, n_features, thresholds, chain=False):
    """one tree in LightGBM's numbering: split k turns a leaf into internal node k, whose left child keeps that leaf and whose
    right child is the new leaf k + 1 (chain: always split the newest leaf, depth n_leaves - 1)"""
    left, right, parent_of_leaf = [], [], {0: None}
    for k in range(n_leaves - 1):
        j = k if chain else int(rng.choice(list(parent_of_leaf)))
        p = parent_of_leaf.pop(j)
        if p is not None:
            node, side = p
            (left if side == 0 else right)[node] = k
        left.append(-1 - j)
        right.append(-1 - (k + 1))
        parent_of_leaf[j] = (k, 0)
        parent_of_leaf[k + 1] = (k, 1)
    feats = [int(rng.integers(0, n_features)) for _ in range(n_leaves - 1)]
    thr = [float(rng.choice(thresholds)) for _ in range(n_leaves - 1)]
    leaves = [float(rng.normal(0, 0.2)) for _ in range(n_leaves)]
    return feats, thr, left, right, leaves


def write_model(feature_names, trees, blank_lines=2):
    """LightGBM model text as the reference reads it: trees = (split_feature, threshold, left_child, right_child, leaf_value)"""
    out = ["tree", "version=v3", "num_class=1", f"max_feature_idx={len(feature_names) - 1}", "objective=lambdarank",
           "feature_names=" + " ".join(feature_names), ""]
    for i, (f, th, lc, rc, lv) in enumerate(trees):
        out += [f"Tree={i}", f"num_leaves={len(lv)}", "split_feature=" + " ".join(map(str, f)),
                "threshold=" + " ".join(repr(x) for x in th), "decision_type=" + " ".join("2" for _ in f),
                "left_child=" + " ".join(map(str, lc)), "right_child=" + " ".join(map(str, rc)),
                "leaf_value=" + " ".join(repr(x) for x in lv), "shrinkage=0.1"] + [""] * blank_lines
    out += ["end of trees", "", "feature_importances:", ""]
    return "\n".join(out)


def random_model(rng, n_trees, leaves, feature_names=None, chain_every=0, thresholds=None):
    """a seeded synthetic model: `leaves` an int or (lo, hi) range of leaf counts; every chain_every-th tree a chain"""
    names = feature_names or [snake_case(n) for n in SIGNAL_ENUM]
    if thresholds is None:
        thresholds = [float(x) for x in rng.normal(0, 1, 64)] + [0.0, -0.0, 1.0, 0.5]
    trees = []
    for t in range(n_trees):
        nl = leaves if isinstance(leaves, int) else int(rng.integers(leaves[0], leaves[1] + 1))
        trees.append(lightgbm_tree(rng, nl, len(names), thresholds, chain=bool(chain_every) and t % chain_every == 0))
    return write_model(names, trees), thresholds


def random_rows(rng, n, thresholds, absent=0.3):
    """feature rows: normals, exact thresholds (the <= edge), +-0.0, NaN, +-inf, absent signals (0.0)"""
    import numpy as np
    X = rng.normal(0, 1, (n, len(SIGNAL_ENUM)))
    pick = rng.random(X.shape)
    th = np.asarray(thresholds)
    X = np.where(pick < 0.25, th[rng.integers(0, th.size, X.shape)], X)
    specials = np.array([0.0, -0.0, np.nan, np.inf, -np.inf])
    X = np.where((pick >= 0.25) & (pick < 0.3), specials[rng.integers(0, specials.size, X.shape)], X)
    X = np.where((pick >= 0.3) & (pick < 0.3 + absent), 0.0, X)
    return X


SIMPLE_FEATURES = {"Bm25BacklinkText": 85.7750244140625, "Bm25CleanBody": 67.41311645507812, "IdfSumDomain": 43.332096099853516,
                   "IdfSumSite": 61.47410202026367, "Bm25StemmedCleanBody": 65.94627380371094, "Bm25Title": 59.817813873291016,
                   "IdfSumUrl": 57.07925033569336, "FetchTimeMs": 0.023255813953488372, "HostCentrality": 0.017958538,
                   "PageCentrality": 0.008253236, "Region": 0.16622349570454012, "TrackerScore": 0.07692307692307693,
                   "UrlDigits": 0.25, "UrlSlashes": 0.3333333333333333}
SIMPLE_BITS = 0x3FF0CF2FF026E69A   # 1.0505828267036237


def simple_row():
    """the features of the reference's `simple` test (lambdamart.rs:320-388); the ones it sets to 0.0 are 0.0 here too"""
    row = [0.0] * len(SIGNAL_ENUM)
    for k, v in SIMPLE_FEATURES.items():
        row[SIGNAL_ENUM.index(k)] = v
    return row
