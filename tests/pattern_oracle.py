"""A plain restatement of Stract's pattern queries and optic rules over per-document token lists, for the tests (it does not
use the library).

  NormalPatternScorer    core/src/query/pattern_query/scorer.rs:203-339, intersection_with_slop :371-409
  pattern_scorer         core/src/query/pattern_query/weight.rs:121-226 (the four branches)
  optic rules            core/src/query/optic.rs:50-169 (rules, as_multiple_tantivy), computer/mod.rs:267-277,471-497 (boosts)

A field is a list of documents, each a list of token ids (position = index).  Parts are "T" (term), "*" (wildcard) and "|"
(anchor); terms are token ids, None for a token the segment does not hold.  `counts[d]` is the token-count fast field (None:
missing)."""
import numpy as np

U32_MAX = 0xFFFFFFFF


def intersection_with_slop(left, right, slop):
    """scorer.rs:371-409, the sequential walk as written."""
    li = ri = 0
    out = []
    while li < len(left) and ri < len(right):
        lv, rv = left[li], right[ri]
        rs = max(rv - slop, 0)
        if lv < rs:
            li += 1
        elif rs <= lv <= rv:
            while li + 1 < len(left):
                if left[li + 1] > rv:
                    break
                li += 1
            out.append(rv)
            ri += 1
        elif lv > rv:
            ri += 1
    return out


def positions(doc_tokens, term):
    return [i for i, t in enumerate(doc_tokens) if t == term]


def normal_pattern_match(doc_tokens, parts, terms, num_tokens):
    """NormalPatternScorer::pattern_match for one candidate document (it holds every term)."""
    return normal_pattern_match_pos([positions(doc_tokens, t) for t in terms], parts, num_tokens)


def normal_pattern_match_pos(pos, parts, num_tokens):
    """The same from the positions of every pattern term (pos[j]: ascending positions of term j in the document)."""
    if len(pos) == 1 and all(p == "T" for p in parts):
        return True                                         # term_freq > 0
    left = list(pos[0])
    n = len(left)
    cur, slop = 0, 1
    for i, p in enumerate(parts):
        if p == "T":
            if cur == 0:
                cur = 1
                continue
            left = intersection_with_slop(left, list(pos[cur]), slop)
            n = len(left)
            slop = 1
            if n == 0:
                return False
            cur += 1
        elif p == "*":
            slop = U32_MAX
        elif i == 0:
            if left and left[0] != 0:
                return False
        elif i == len(parts) - 1:
            right = list(pos[-1])
            if right and right[-1] != ((num_tokens - 1) & 0xFFFFFFFFFFFFFFFF) & U32_MAX:
                return False
    return n > 0


def pattern_docs(field_docs, parts, terms, counts=None):
    """PatternWeight::pattern_scorer + the scorer's docset: the sorted matching documents."""
    n_docs = len(field_docs)
    if not parts:
        return []
    if not terms and "*" in parts:
        return list(range(n_docs))
    if not terms:
        return [d for d in range(n_docs) if (counts[d] or 0) == 0]
    if any(t is None for t in terms):
        return []
    out = []
    for d, toks in enumerate(field_docs):
        if all(t in toks for t in terms):
            nt = None if counts is None else counts[d]
            if "|" in parts and nt is None and not (len(terms) == 1 and all(p == "T" for p in parts)):
                raise ValueError(f"doc {d}: NormalPatternScorer unwraps a missing token count")
            if normal_pattern_match(toks, parts, terms, 0 if nt is None else nt):
                out.append(d)
    return out


def rule_docs(blocks, matching_docs):
    """A rule: OR over its non-empty blocks of the AND of their matchings; None when no block is left (no rule)."""
    blocks = [b for b in blocks if b]
    if not blocks:
        return None
    out = set()
    for b in blocks:
        s = set(matching_docs(b[0]))
        for m in b[1:]:
            s &= set(matching_docs(m))
        out |= s
    return out


def boost_factor(doc, rules):
    """SignalComputer::boosts: rules = [(docset, boost f64)] in rule order."""
    down = up = 0.0
    for docs, b in rules:
        if doc in docs:
            if b < 0.0:
                down += abs(b)
            else:
                up += b
    return 1.0 / (1.0 + (down - up)) if down > up else up - down + 1.0


def optic_topk(candidates, k, rules=(), exclude=None, require=None):
    """The recall stage with docset rules: `candidates` = [(doc, total)] of every candidate without optics (the multi-field
    oracle's totals), filtered by exclude / require, multiplied by the boost factor, top-k by (total desc, doc asc)."""
    out = []
    for d, t in candidates:
        d = int(d)
        if exclude is not None and d in exclude:
            continue
        if require is not None and d not in require:
            continue
        if rules:
            t = float(np.float64(t) * np.float64(boost_factor(d, rules)))
        out.append((t, d))
    out.sort(key=lambda x: (-x[0], x[1]))
    return out[:k]
