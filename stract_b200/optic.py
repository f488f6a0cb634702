"""Optic rules on the device: the host half of Stract's optics (optics/src/lib.rs) and of their recall-stage use
(core/src/query/optic.rs, core/src/query/mod.rs:129-137, core/src/ranking/computer/mod.rs:267-277,471-497).

The optic text parser and Stract's tokenizers are not part of this library: callers hand over parsed structures and a resolver
`resolve(field, raw_text, exact)` that returns the term ordinals of raw_text's tokens in that field's segment (ABSENT_TERM for
a token the segment lacks); with exact=True it returns [the ordinal of raw_text as one untokenised term] (the no-tokenizer
lookup of FastSiteDomainPatternWeight).  The Domain -> Site rewrite asks `root_domain(text)` (Url::root_domain of
"https://" + text, or None).

compile_optics builds every distinct matching's docset once per segment, so queries that share an optic share its bitmaps."""
from .bm25 import (ABSENT_TERM, MAX_OPTIC_RULES, MAX_QUERY_TERMS, PART_ANCHOR, PART_TERM, PART_WILDCARD, Docset, OpticTables,
                   pattern_docsets)

TYPE_PREFIX = "$"   # schema_org::TYPE_PREFIX (core/src/webpage/schema_org/mod.rs:27-30)

# MatchLocation -> text field (optic.rs:179-235)
LOCATION_FIELD = {"Site": "UrlForSiteOperator", "Url": "Url", "Domain": "Domain", "Title": "Title", "Description": "Description",
                  "Content": "CleanBody", "MicroformatTag": "MicroformatTags", "Schema": "FlattenedSchemaOrgJson"}


class PatternPart:
    """PatternPart::Raw(text) / Wildcard / Anchor."""
    __slots__ = ("kind", "text")

    def __init__(self, kind, text=None):
        self.kind, self.text = kind, text

    @classmethod
    def raw(cls, text):
        return cls("raw", text)

    def __eq__(self, o):
        return isinstance(o, PatternPart) and (self.kind, self.text) == (o.kind, o.text)

    def __hash__(self):
        return hash((self.kind, self.text))

    def __repr__(self):
        return {"raw": repr(self.text), "wildcard": "*", "anchor": "|"}[self.kind]


PatternPart.WILDCARD = PatternPart("wildcard")
PatternPart.ANCHOR = PatternPart("anchor")


def parse_pattern(s):
    """The pattern syntax of optics (`|` anchor, `*` wildcard, everything else raw text) into parts; a convenience for tests
    and tools, equal to what the optics parser produces for a pattern string."""
    parts, cur = [], ""
    for ch in s:
        if ch in "|*":
            if cur:
                parts.append(PatternPart.raw(cur)); cur = ""
            parts.append(PatternPart.ANCHOR if ch == "|" else PatternPart.WILDCARD)
        else:
            cur += ch
    if cur:
        parts.append(PatternPart.raw(cur))
    return parts


class Matching:
    def __init__(self, pattern, location):
        self.pattern = parse_pattern(pattern) if isinstance(pattern, str) else list(pattern)
        self.location = location


class Action:
    """Boost(n) / Downrank(n) / Discard (optics lib.rs:334-338); a rule without an action is Boost(0) (lib.rs:130)."""

    def __init__(self, kind, value=0):
        self.kind, self.value = kind, int(value)

    @classmethod
    def boost(cls, n):
        return cls("boost", n)

    @classmethod
    def downrank(cls, n):
        return cls("downrank", n)


Action.DISCARD = Action("discard")


class Rule:
    def __init__(self, matches, action=None):
        self.matches = [list(block) for block in matches]   # OR over blocks of the AND of their matchings
        self.action = Action.boost(0) if action is None else action


class HostRankings:
    def __init__(self, liked=(), disliked=(), blocked=()):
        self.liked, self.disliked, self.blocked = list(liked), list(disliked), list(blocked)

    def rules(self):
        """HostRankings::rules (optics lib.rs:531-556): a Discard rule with one Site("|host|") block per blocked host, "www."
        stripped."""
        blocks = [[Matching([PatternPart.ANCHOR, PatternPart.raw(h[4:] if h.startswith("www.") else h), PatternPart.ANCHOR], "Site")]
                  for h in self.blocked]
        return Rule(blocks, Action.DISCARD)


class Optic:
    def __init__(self, rules=(), discard_non_matching=False, host_rankings=None):
        self.rules = list(rules)
        self.discard_non_matching = bool(discard_non_matching)
        self.host_rankings = host_rankings or HostRankings()


def can_optimize_site_domain(parts, field):
    """pattern_query/mod.rs:166-175: |raw ... raw| on the Site or Domain field reads one untokenised term."""
    return (len(parts) >= 2 and parts[0].kind == "anchor" and parts[-1].kind == "anchor"
            and all(p.kind == "raw" for p in parts[1:-1]) and field in ("UrlForSiteOperator", "Domain"))


def matching_target(m, root_domain=None):
    """Matching::as_tantivy (optic.rs:179-235): the (field, parts) of the PatternQuery a matching becomes, with the Domain ->
    Site rewrite (a |raw| domain that is not its own root domain) and the Schema prefix on the first raw part."""
    if m.location == "Domain" and len(m.pattern) == 3 and m.pattern[0].kind == "anchor" and m.pattern[2].kind == "anchor" \
            and m.pattern[1].kind == "raw" and root_domain is not None:
        real = root_domain(m.pattern[1].text)
        if real is not None and real != m.pattern[1].text:
            return "UrlForSiteOperator", list(m.pattern)
    if m.location == "Schema":
        parts = list(m.pattern)
        for i, p in enumerate(parts):
            if p.kind == "raw":
                parts[i] = PatternPart.raw(TYPE_PREFIX + p.text)
                break
        return "FlattenedSchemaOrgJson", parts
    return LOCATION_FIELD[m.location], list(m.pattern)


def pattern_row(field, parts, resolve):
    """PatternQuery::new (pattern_query/mod.rs:51-128): ("postings", ordinal) for the site / domain fast path, else
    ("pattern", (part kinds, term ordinals)) with every raw part tokenised."""
    if can_optimize_site_domain(parts, field):
        text = "".join(p.text for p in parts if p.kind == "raw")
        return "postings", int(resolve(field, text, True)[0])
    kinds, ords = [], []
    for p in parts:
        if p.kind == "raw":
            toks = [int(t) for t in resolve(field, p.text, False)]
            kinds += [PART_TERM] * len(toks); ords += toks
        else:
            kinds.append(PART_WILDCARD if p.kind == "wildcard" else PART_ANCHOR)
    if len(ords) > MAX_QUERY_TERMS:
        raise ValueError(f"pattern {parts!r} on {field} has {len(ords)} terms; at most {MAX_QUERY_TERMS}")
    return "pattern", (tuple(kinds), tuple(ords))


def searchable_rule(rule):
    """Rule::as_searchable_rule (optic.rs:104-169): the rule's blocks without the empty ones (None: no rule at all) and its
    boost (Boost b -> b, Downrank b -> -b as f64, Discard -> 0)."""
    blocks = [b for b in rule.matches if b]
    if not blocks:
        return None
    boost = {"boost": float(rule.action.value), "downrank": float(rule.action.value) * -1.0, "discard": 0.0}[rule.action.kind]
    return blocks, boost


def boost_rules(optics):
    """SignalComputer's rules (computer/mod.rs:267-277): Boost / Downrank with b != 0, over the optics in order."""
    return [r for o in optics for r in o.rules if r.action.kind != "discard" and r.action.value != 0]


class _Builder:
    """The docsets of one segment, each distinct matching / rule built once."""

    def __init__(self, fields, resolve, root_domain):
        self.fields, self.resolve, self.root_domain = fields, resolve, root_domain
        self.docsets, self.index = [], {}

    def _add(self, key, make):
        if key not in self.index:
            self.index[key] = len(self.docsets)
            self.docsets.append(make())
        return self.index[key]

    def prepare(self, matchings):
        """Builds the docsets of all distinct matchings, one pattern batch per field."""
        pending = {}
        for m in matchings:
            field, parts = matching_target(m, self.root_domain)
            kind, row = pattern_row(field, parts, self.resolve)
            key = ("m", field, kind, row)
            if key in self.index:
                continue
            if kind == "postings":
                self._add(key, lambda: Docset.from_postings(self.fields[field], row))
            else:
                pending.setdefault(field, {}).setdefault(key, row)
        for field, rows in pending.items():
            keys = list(rows)
            out = pattern_docsets(self.fields[field], [(list(rows[k][0]), list(rows[k][1])) for k in keys])
            for k, d in zip(keys, out):
                self._add(k, lambda d=d: d)

    def matching(self, m):
        field, parts = matching_target(m, self.root_domain)
        kind, row = pattern_row(field, parts, self.resolve)
        key = ("m", field, kind, row)
        if key not in self.index:
            self.prepare([m])
        return self.index[key]

    def combine(self, op, idx):
        idx = list(idx)
        if len(idx) == 1:
            return idx[0]
        return self._add((op, tuple(idx)), lambda: Docset.combine(op, [self.docsets[i] for i in idx]))

    def rule(self, blocks):
        return self.combine("or", [self.combine("and", [self.matching(m) for m in b]) for b in blocks])

    def empty(self):
        any_reader = next(iter(self.fields.values()))
        return self._add(("empty",), lambda: Docset.from_postings(any_reader, ABSENT_TERM))


def compile_optics(fields, query_optics, resolve, root_domain=None):
    """OpticTables for a batch: `fields` = {text field name: SegmentReader} of one segment, `query_optics[q]` = the optics of
    query q (several optics nest: their filters AND).  Per query:
      rules    SignalComputer's boost rules, (docset, +-b) in rule order;
      exclude  the OR of every optic's Discard rules and blocked hosts (MustNot);
      require  the AND over the DiscardNonMatching optics of the OR of their non-Discard rules, Boost(0) ones included (Must)."""
    B = _Builder(fields, resolve, root_domain)
    every = [m for optics in query_optics for o in optics for r in list(o.rules) + [o.host_rankings.rules()] for b in r.matches for m in b]
    B.prepare(every)
    rules, exclude, require = [], [], []
    for optics in query_optics:
        rq = []
        for r in boost_rules(optics):
            sr = searchable_rule(r)
            if sr is not None:
                rq.append((B.rule(sr[0]), sr[1]))
        if len(rq) > MAX_OPTIC_RULES:
            raise ValueError(f"a query has {len(rq)} optic boost rules; at most {MAX_OPTIC_RULES}")
        rules.append(rq)
        ex, req = [], []
        for o in optics:
            for r in [r for r in o.rules if r.action.kind == "discard"] + [o.host_rankings.rules()]:
                sr = searchable_rule(r)
                if sr is not None:
                    ex.append(B.rule(sr[0]))
            if o.discard_non_matching:
                keep = [searchable_rule(r) for r in o.rules if r.action.kind != "discard"]
                keep = [B.rule(sr[0]) for sr in keep if sr is not None]
                req.append(B.combine("or", keep) if keep else B.empty())
        exclude.append(B.combine("or", ex) if ex else None)
        require.append(B.combine("and", req) if req else None)
    return OpticTables(B.docsets, rules, exclude, require)
