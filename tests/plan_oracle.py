"""Plain restatement of a compiled plan's docset: BooleanWeight (tantivy/src/query/boolean_query/boolean_weight.rs:107-180)
over document sets, with scoring disabled.  A program is the post-order node list of sb200_recall_plan_batch; `leaf(node)`
gives a leaf's document set."""
from stract_b200.bm25 import ABSENT_TERM, PLAN_BOOL, PLAN_EMPTY, PLAN_MUST, PLAN_MUST_NOT, PLAN_PHRASE, PLAN_SHOULD, PLAN_TERM


def boolean(clauses):
    """clauses: [(occur, set)] -> the BooleanWeight docset"""
    if not clauses:
        return set()
    if len(clauses) == 1:
        occ, s = clauses[0]
        return set() if occ == PLAN_MUST_NOT else set(s)
    must = [s for o, s in clauses if o == PLAN_MUST]
    should = [s for o, s in clauses if o == PLAN_SHOULD]
    nots = set().union(*[s for o, s in clauses if o == PLAN_MUST_NOT])
    if must:
        out = set.intersection(*[set(s) for s in must])
    elif should:
        out = set().union(*should)
    else:
        return set()
    return out - nots


def program_docs(prog, postings, phrases=None):
    """postings[segment][ordinal] -> iterable of docs; phrases[row] -> the docs where that phrase exists (phrase_exists_docs)"""
    st = []
    for kind, occ, nc, seg, arg in prog:
        if kind == PLAN_TERM:
            v = set() if arg == ABSENT_TERM else set(int(d) for d in postings[seg][arg])
        elif kind == PLAN_PHRASE:
            v = set(phrases[arg])
        elif kind == PLAN_EMPTY:
            v = set()
        elif kind == PLAN_BOOL:
            kids = st[len(st) - nc:] if nc else []
            del st[len(st) - nc:]
            v = boolean(kids)
        else:
            raise ValueError(f"kind {kind}")
        st.append((occ, v))
    assert len(st) == 1
    return sorted(st[0][1])


def phrase_exists_docs(index, terms, offsets, slop):
    """Documents where PhraseScorer::phrase_exists holds (scoring disabled), by tests/phrase_oracle.py; a None term = absent."""
    import phrase_oracle as O
    n = index["fieldnorm_ids"].size
    hits = O.phrase_search(index, terms, offsets, slop, False, 1.0, [1.0] * 256, n)
    return sorted(int(d) for _, d in hits)
