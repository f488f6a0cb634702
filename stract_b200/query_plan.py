"""Host mirror of Stract's query plan (core/src/query/plan/): the recall docset a parsed query compiles to.

`initial` builds plan::Node from the parser's terms (plan/mod.rs:235-300): the terms are ANDed, each simple term an OR over the
searchable fields plus, with <= MAX_TERMS_FOR_NGRAM_LOOKUPS terms, its 2- and 3-term compounds over the compound-searchable
fields.  `into_query` is Node::into_query (node.rs:98-103): optimise (Deduplicate, then DistributiveLaw), the non-compacted
query, `compact`, `deduplicate`.  `compile_plans` applies as_tantivy's leaf choice (plan/mod.rs:137-200) through a caller
resolver and emits the post-order programs of sb200_recall_plan_batch.

DistributiveLaw collects the common children of two ORs through a HashSet, so the clause order of its output is not fixed
upstream.  The docset does not depend on clause order, so this mirror keeps the order of first appearance and its tests
compare with the reference tests as sets where the order is free.  Tokenising and the term -> ordinal lookup belong to the
caller (`resolver`), as in stract_b200.optic."""
from dataclasses import dataclass

from .bm25 import (ABSENT_TERM, PLAN_BOOL, PLAN_EMPTY, PLAN_MUST, PLAN_MUST_NOT, PLAN_PHRASE, PLAN_SHOULD, PLAN_TERM, RecallPlan)

MAX_TERMS_FOR_NGRAM_LOOKUPS = 16
MUST, SHOULD, MUST_NOT = PLAN_MUST, PLAN_SHOULD, PLAN_MUST_NOT


@dataclass(frozen=True)
class Term:
    """plan::Term: `text` is ("simple", str) or ("phrase", tuple of words), `field` a text field name."""
    text: tuple
    field: str


@dataclass
class Schema:
    """The text fields in TextFieldEnum order and their flags (schema/text_field.rs)."""
    searchable: list
    phrase_searchable: set
    compound_searchable: set
    positions: set


class Node:
    """plan::Node: ("term", Term) | ("and", a, b) | ("or", a, b) | ("not", a).  And / Or compare commutatively (node.rs:34-45)."""
    __slots__ = ("op", "a", "b")

    def __init__(self, op, a, b=None):
        self.op, self.a, self.b = op, a, b

    def __eq__(self, o):
        if not isinstance(o, Node) or self.op != o.op:
            return False
        if self.op in ("and", "or"):
            return (self.a == o.a and self.b == o.b) or (self.a == o.b and self.b == o.a)
        return self.a == o.a

    def __hash__(self):
        return hash(self.op) if self.op in ("and", "or") else hash((self.op, self.a))

    def __repr__(self):
        return f"{self.a.field}:{self.a.text[1]}" if self.op == "term" else f"{self.op}({self.a!r}, {self.b!r})" if self.b is not None else f"not({self.a!r})"

    def and_(self, o):
        return Node("and", self, o)

    def or_(self, o):
        return Node("or", self, o)


def term(text, field):
    return Node("term", Term(text, field))


def _reduce(nodes, op):
    out = None
    for n in nodes:
        out = n if out is None else Node(op, out, n)
    return out


def from_term(t, schema):
    """Node::from_term for every parser term kind (node.rs:105-171): ("simple", s), ("phrase", words), ("site", s),
    ("linkto", s), ("title" | "body" | "url", ("simple", s) | ("phrase", words)), ("exacturl", s), ("bang", prefix, bang), ("not", t)."""
    kind = t[0]
    if kind == "simple":
        return _reduce([term(("simple", t[1]), f) for f in schema.searchable], "or")
    if kind == "phrase":
        return _reduce([term(("phrase", tuple(t[1])), f) for f in schema.searchable if f in schema.phrase_searchable], "or")
    if kind == "site":
        return term(("simple", t[1]), "UrlForSiteOperator")
    if kind == "linkto":
        return term(("simple", t[1]), "Links")
    if kind in ("title", "body", "url"):
        sop = t[1]
        return term(sop if sop[0] == "simple" else ("phrase", tuple(sop[1])), {"title": "Title", "body": "AllBody", "url": "Url"}[kind])
    if kind == "exacturl":
        return term(("simple", t[1]), "UrlNoTokenizer")
    if kind == "bang":
        return _reduce([term(("simple", t[1] + t[2]), f) for f in schema.searchable], "or")
    if kind == "not":
        return Node("not", from_term(t[1], schema))
    raise ValueError(f"unknown term kind {kind!r}")


def sliding_window(window_size, i):
    """plan/mod.rs:224-233"""
    return [(max(i + o - window_size, 0), i + o) for o in range(window_size + 1) if max(i + o - window_size, 0) < i + o]


def initial(terms, schema):
    """plan::initial (plan/mod.rs:235-300); None for no terms"""
    nodes = []
    augment = len(terms) <= MAX_TERMS_FOR_NGRAM_LOOKUPS
    for i, t in enumerate(terms):
        adjacent = []
        if augment and t[0] == "simple":
            for w in (2, 3):
                for start, end in sliding_window(w, i):
                    comp = [terms[k][1] for k in range(start, end + 1) if k < len(terms) and terms[k][0] == "simple"]
                    if comp:
                        adjacent.append(comp)
        node = from_term(t, schema)
        adj = _reduce([term(("simple", "".join(c)), f) for c in adjacent for f in schema.searchable if f in schema.compound_searchable], "or")
        nodes.append(node.or_(adj) if adj is not None else node)
    return _reduce(nodes, "and")


def _or_children(n):
    if n.op == "or":
        out = _or_children(n.a)
        for c in _or_children(n.b):
            if c not in out:
                out.append(c)
        return out
    return [n]


def _prune(n, child):
    if n.op == "or":
        if n.a == child:
            return n.b
        if n.b == child:
            return n.a
        return Node("or", _prune(n.a, child), _prune(n.b, child))
    return n


def _dedup(n):
    if n.op == "term":
        return n
    if n.op == "not":
        return Node("not", _dedup(n.a))
    a, b = _dedup(n.a), _dedup(n.b)
    return a if a == b else Node(n.op, a, b)


def _distribute(n):
    if n.op == "term":
        return n
    if n.op == "not":
        return Node("not", _distribute(n.a))
    a, b = _distribute(n.a), _distribute(n.b)
    if n.op == "or" or a.op != "or" or b.op != "or":
        return Node(n.op, a, b)
    rc = _or_children(b)
    common = [c for c in _or_children(a) if c in rc]
    if not common:
        return Node("and", a, b)
    for c in common:
        a, b = _prune(a, c), _prune(b, c)
    return Node("or", Node("and", a, b), _reduce(common, "or"))


def optimise(n):
    """Node::optimise: Deduplicate, then DistributiveLaw"""
    return _distribute(_dedup(n))


def compose(left, right):
    """Occur::compose (plan/mod.rs:33-43)"""
    if left == SHOULD:
        return right
    if left == MUST:
        return MUST_NOT if right == MUST_NOT else MUST
    return MUST if right == MUST_NOT else MUST_NOT


# a Query is ("term", Term) or ("bool", [(occur, Query), ...])
def _non_compacted(n):
    if n.op == "term":
        return ("term", n.a)
    if n.op == "not":
        return ("bool", [(MUST_NOT, _non_compacted(n.a))])
    occ = MUST if n.op == "and" else SHOULD
    return ("bool", [(occ, _non_compacted(n.a)), (occ, _non_compacted(n.b))])


def compact(q):
    """Query::compact (plan/mod.rs:81-117)"""
    if q[0] == "term":
        return q
    out = []
    for occ, sub in q[1]:
        sub = compact(sub)
        if sub[0] == "bool" and all(o == occ for o, _ in sub[1]):
            out.extend(sub[1])
        elif sub[0] == "bool" and len(sub[1]) == 1:
            out.append((compose(occ, sub[1][0][0]), sub[1][0][1]))
        else:
            out.append((occ, sub))
    return ("bool", out)


def _freeze(q):
    return q if q[0] == "term" else ("bool", tuple((o, _freeze(s)) for o, s in q[1]))


def deduplicate(q):
    """Query::deduplicate (plan/mod.rs:119-131): unique clauses, first occurrence kept"""
    if q[0] == "term":
        return q
    seen, out = set(), []
    for occ, sub in q[1]:
        sub = deduplicate(sub)
        key = (occ, _freeze(sub))
        if key not in seen:
            seen.add(key)
            out.append((occ, sub))
    return ("bool", out)


def into_query(n):
    return deduplicate(compact(_non_compacted(optimise(n))))


def parse(terms, schema, safe_search=False):
    """Query::parse's plan (query/mod.rs:106-122): initial, the safe-search Not, into_query"""
    plan = initial(terms, schema)
    if plan is None:
        raise ValueError("no terms")
    if safe_search:
        # safety_classifier::Label::NSFW.to_string() is "NSFW"; SafetyClassification's Identity tokenizer keeps its case
        plan = plan.and_(Node("not", term(("simple", "NSFW"), "SafetyClassification")))
    return into_query(plan)


def compile_query(q, field_index, resolver, schema, phrases=None):
    """as_tantivy (plan/mod.rs:137-200) into a post-order program.  resolver(field, text) -> the ordinals of the text's tokens
    in that field (ABSENT_TERM for a token the segment lacks), or None when the field is not in the schema.  A PhraseQuery leaf
    appends its row (ordinals, offsets 0, 1, 2, ..., slop 0) to `phrases` and refers to it.  Returns None for a dropped clause
    (a phrase with no tokens)."""
    if phrases is None:
        phrases = []
    if q[0] == "bool":
        prog, n = [], 0
        for occ, sub in q[1]:
            p = compile_query(sub, field_index, resolver, schema, phrases)
            if p is None:
                continue
            k, _, nc, sg, arg = p[-1]
            prog += p[:-1] + [(k, occ, nc, sg, arg)]
            n += 1
        return prog + [(PLAN_BOOL, MUST, n, 0, 0)]
    t = q[1]
    words = t.text[1] if t.text[0] == "simple" else " ".join(t.text[1])
    toks = resolver(t.field, words) if t.field in field_index else None
    toks = [] if toks is None else list(toks)
    seg = field_index.get(t.field, 0)
    if t.text[0] == "phrase" and not toks:
        return None
    if len(toks) == 1:
        return [(PLAN_TERM, MUST, 0, seg, toks[0])]
    if not toks:
        return [(PLAN_EMPTY, MUST, 0, 0, 0)]
    if t.text[0] == "phrase" or t.field in schema.positions:
        phrases.append((toks, None, 0))
        return [(PLAN_PHRASE, MUST, 0, seg, len(phrases) - 1)]
    return [(PLAN_TERM, MUST, 0, seg, o) for o in toks] + [(PLAN_BOOL, MUST, len(toks), 0, 0)]


def compile_plans(queries, segments, resolver, schema):
    """queries: per query its compiled Query (into_query / parse); segments: {field name: SegmentReader}.  -> RecallPlan"""
    names = list(segments)
    index = {n: i for i, n in enumerate(names)}
    progs, phrases = [], []
    for q in queries:
        p = compile_query(q, index, resolver, schema, phrases)
        progs.append(p if p is not None else [(PLAN_EMPTY, MUST, 0, 0, 0)])
    return RecallPlan([segments[n] for n in names], progs, phrases)


__all__ = ["ABSENT_TERM", "MUST", "SHOULD", "MUST_NOT", "Node", "Schema", "Term", "compact", "compile_plans", "compile_query", "compose",
           "deduplicate", "from_term", "initial", "into_query", "optimise", "parse", "sliding_window", "term"]
