"""The query-plan mirror (stract_b200/query_plan.py) against the reference's plan tests (plan/mod.rs:351-441, node.rs), and
the BooleanWeight restatement (plan_oracle.py) on a hand-made case for every rule.  The end-to-end tests of query/mod.rs
(not_query, site_query, phrase_query, match_compound_words, mix_phrase_term_query, ...) index real pages through Stract's
tokenizers and are not pinned here."""
from stract_b200 import query_plan as QP
from stract_b200.bm25 import ABSENT_TERM, PLAN_BOOL, PLAN_EMPTY, PLAN_PHRASE, PLAN_TERM
import plan_oracle as PO

M, S, N = QP.MUST, QP.SHOULD, QP.MUST_NOT
SCHEMA = QP.Schema(["Title", "AllBody", "Url"], {"Title", "AllBody"}, {"Title"}, set())


def T(text, field="Title"):
    return QP.term(("simple", text), field)


def test_sliding_window():
    assert QP.sliding_window(3, 3) == [(0, 3), (1, 4), (2, 5), (3, 6)]
    assert QP.sliding_window(2, 3) == [(1, 3), (2, 4), (3, 5)]
    assert QP.sliding_window(2, 0) == [(0, 1), (0, 2)]


def test_compact():
    assert QP.compact(("bool", [])) == ("bool", [])
    node = T("foo", "Title").or_(T("foo", "AllBody")).and_(T("bar", "Title").or_(T("bar", "AllBody")))
    got = QP.compact(QP.into_query(node))                  # query.into_query().compact(), as the reference test
    want = ("bool", [(M, ("bool", [(S, ("term", QP.Term(("simple", "foo"), "Title"))), (S, ("term", QP.Term(("simple", "foo"), "AllBody")))])),
                     (M, ("bool", [(S, ("term", QP.Term(("simple", "bar"), "Title"))), (S, ("term", QP.Term(("simple", "bar"), "AllBody")))]))])
    assert got == want


def test_optimisation():
    a, b, c, d, e, f = (T(x) for x in "abcdef")
    assert QP.optimise(a.or_(b).and_(a.or_(c))) == a.or_(b.and_(c))
    assert QP.optimise(a.or_(b).and_(c.or_(d))) == a.or_(b).and_(c.or_(d))
    got = QP.optimise(a.or_(b).or_(c).or_(d).and_(e.or_(f).or_(c).or_(d)))
    assert got.op == "or" and got.a == a.or_(b).and_(e.or_(f))
    assert set(QP._or_children(got.b)) == {c, d}          # the common children come out of a HashSet upstream: any order
    assert QP.optimise(a.or_(a).or_(a).or_(a).and_(a.or_(a).or_(a).or_(a))) == a
    assert QP.optimise(a.or_(b).and_(a.or_(c.and_(a)))) == a.or_(b.and_(c.and_(a)))


def test_initial_compounds_and_fields():
    q = QP.initial([("simple", "x"), ("simple", "y")], SCHEMA)
    assert q.op == "and"
    kids = QP._or_children(q.a)
    assert T("x", "Title") in kids and T("x", "Url") in kids and T("xy", "Title") in kids and T("xy", "Url") not in kids
    assert QP.from_term(("site", "a.com"), SCHEMA) == T("a.com", "UrlForSiteOperator")
    assert QP.from_term(("phrase", ["p", "q"]), SCHEMA) == QP.term(("phrase", ("p", "q")), "Title").or_(QP.term(("phrase", ("p", "q")), "AllBody"))
    assert QP.compose(M, N) == N and QP.compose(N, N) == M and QP.compose(S, N) == N


def test_boolean_rules():
    A, B = {1, 2, 3}, {3, 4}
    assert PO.boolean([]) == set()
    assert PO.boolean([(N, A)]) == set()
    assert PO.boolean([(S, A)]) == A
    assert PO.boolean([(M, A), (S, B)]) == A                 # Should is ignored when a Must exists
    assert PO.boolean([(S, A), (S, B), (N, {1})]) == {2, 3, 4}
    assert PO.boolean([(N, A), (N, B)]) == set()
    assert PO.boolean([(M, A), (M, B)]) == {3}


def test_leaf_choice_and_safe_search():
    idx = {"Title": 0, "AllBody": 1}
    res = {"a": [5], "": [], "ab": [1, 2], "zz": [ABSENT_TERM]}
    r = lambda field, text: res.get(text, [])
    simple0 = ("term", QP.Term(("simple", ""), "Title"))
    phrase0 = ("term", QP.Term(("phrase", ()), "Title"))
    assert QP.compile_query(simple0, idx, r, SCHEMA) == [(PLAN_EMPTY, M, 0, 0, 0)]       # kept, matches nothing
    assert QP.compile_query(phrase0, idx, r, SCHEMA) is None                            # dropped
    prog = QP.compile_query(("bool", [(S, simple0), (S, phrase0), (S, ("term", QP.Term(("simple", "a"), "AllBody")))]), idx, r, SCHEMA)
    assert prog == [(PLAN_EMPTY, S, 0, 0, 0), (PLAN_TERM, S, 0, 1, 5), (PLAN_BOOL, M, 2, 0, 0)]
    assert QP.compile_query(("term", QP.Term(("simple", "ab"), "Title")), idx, r, SCHEMA)[-1] == (PLAN_BOOL, M, 2, 0, 0)
    pos = QP.Schema(SCHEMA.searchable, SCHEMA.phrase_searchable, SCHEMA.compound_searchable, {"Title"})
    assert QP.compile_query(("term", QP.Term(("simple", "ab"), "Title")), idx, r, pos)[0][0] == PLAN_PHRASE
    assert QP.compile_query(("term", QP.Term(("simple", "a"), "Links")), idx, r, SCHEMA) == [(PLAN_EMPTY, M, 0, 0, 0)]   # no such field
    post = [[[1, 2, 3], [2]], [[3, 4], [9]]]
    assert PO.program_docs([(PLAN_TERM, M, 0, 0, 0), (PLAN_TERM, M, 0, 0, ABSENT_TERM), (PLAN_BOOL, M, 2, 0, 0)], post) == []
    q = QP.parse([("simple", "a")], SCHEMA, safe_search=True)
    assert q[0] == "bool" and q[1][-1][0] == N and q[1][-1][1][1] == QP.Term(("simple", "NSFW"), "SafetyClassification")
