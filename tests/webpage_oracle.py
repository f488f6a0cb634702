"""A plain restatement of what LocalRecallRankingWebpage::new takes from Stract's SignalComputer (core/src/ranking/computer/,
pipeline/stages/recall.rs:167-220), over per-document postings with positions -- the oracle of sb200_multi_signal_webpages.

A field is {"terms": [{"docs": ascending doc ids, "positions": [absolute positions per doc]} or {"docs", "tfs"}], "ids": fieldnorm
ids}.  Scores follow the reference's operation order: f32 BM25 parts summed in slot order, the f64 sum of the per-field f32 BM25F
sums, coverage in f64, the f32 idf sum, n-gram dampening in f64, then boosts in rule order; min_slop is the reference's
sequential two-cursor walk (stract_b200.ranking_pipeline.min_slop)."""
import numpy as np

from stract_b200.ranking_pipeline import U32_MAX, min_slop

F32 = np.float32
OP_BM25, OP_BM25F, OP_COVERAGE, OP_IDF_SUM, OP_NUMERIC = 0, 1, 2, 3, 4
NO_TERM = 0xFFFFFFFF


def term_maps(field):
    """per term {doc: (tf, positions or None)}"""
    out = []
    for t in field["terms"]:
        if "positions" in t:
            out.append({int(d): (len(p), [int(x) for x in p]) for d, p in zip(t["docs"], t["positions"])})
        else:
            out.append({int(d): (int(tf), None) for d, tf in zip(t["docs"], t["tfs"])})
    return out


class Oracle:
    """`fields` in the computer's field order, `caches` [n_fields][256] f32, `k1`, `coefs` (bm25f coefficient per field, f32),
    `ops` [(kind, field, chain, col, coeff)], `cols` numeric score columns."""

    def __init__(self, fields, caches, k1, coefs, ops, cols):
        self.maps = [term_maps(f) for f in fields]
        self.ids = [np.asarray(f["ids"]) for f in fields]
        self.caches = [np.asarray(c, F32) for c in caches]
        self.k1p1 = F32(F32(k1) + F32(1.0))
        self.coefs = [F32(c) for c in coefs]
        self.ops, self.cols = ops, cols

    def _tf(self, f, ord_, d):
        if ord_ == NO_TERM or ord_ >= len(self.maps[f]):
            return 0, None
        return self.maps[f][ord_].get(d, (0, None))

    def page(self, d, slots, idf, idf_f, rule_slots=(), rules=(), dist=(None, None)):
        """slots: [(field, ord)] text slots in query order; idf / idf_f per slot (f32); rule_slots [(docs set, boost)] in slot
        order, rules [(docs set, boost)] in rule order.  Returns (values, scores, boost, (title slop, body slop))."""
        nf = len(self.maps)
        tf = [self._tf(f, o, d)[0] for f, o in slots]
        n_slots = [sum(1 for f, _ in slots if f == g) for g in range(nf)]
        values, scores = [], []
        hits = 0
        for kind, field, chain, col, _coeff in self.ops:
            sc = 0.0
            if kind == OP_NUMERIC:
                sc = float(self.cols[col][d])
            elif kind == OP_BM25F:
                for g in range(nf):
                    if n_slots[g] == 0:
                        continue
                    norm = self.caches[g][self.ids[g][d]]
                    b = F32(0.0)
                    for x, (f, _o) in enumerate(slots):
                        if f != g:
                            continue
                        part = F32(0.0)
                        if tf[x]:
                            t = F32(F32(tf[x]) * self.coefs[g])
                            part = F32(F32(idf_f[x]) * F32(F32(t * self.k1p1) / F32(t + norm)))
                        b = F32(b + part)
                    sc = sc + float(b)
            elif n_slots[field]:
                xs = [x for x, (f, _o) in enumerate(slots) if f == field]
                if kind == OP_BM25:
                    norm = self.caches[field][self.ids[field][d]]
                    b = F32(0.0)
                    for x in xs:
                        part = F32(0.0)
                        if tf[x]:
                            t = F32(tf[x])
                            part = F32(F32(idf[x]) * F32(F32(t * self.k1p1) / F32(t + norm)))
                        b = F32(b + part)
                    sc = float(b)
                elif kind == OP_COVERAGE:
                    n = 0.0
                    for x in xs:
                        n += 1.0 if tf[x] else 0.0
                    sc = n / float(n_slots[field])
                elif kind == OP_IDF_SUM:
                    b = F32(0.0)
                    for x in xs:
                        if tf[x]:
                            b = F32(b + F32(idf[x]))
                    sc = float(b)
            value = sc
            if chain:
                if chain == 1:
                    hits = 0
                sc = sc * 0.4 ** min(hits, 2)
                if sc > 0.0:
                    hits += 1
            values.append(value)
            scores.append(sc)
        boost = 1.0
        for group in (rule_slots, rules):
            if not group:
                continue
            down = up = 0.0
            for docs, b in group:
                if d in docs:
                    if b < 0.0:
                        down += abs(b)
                    else:
                        up += b
            boost *= 1.0 / (1.0 + (down - up)) if down > up else up - down + 1.0
        slops = []
        for f in dist:
            if f is None:
                slops.append(U32_MAX)
                continue
            lists = []
            for g, o in slots:
                if g == f:
                    t, pos = self._tf(g, o, d)
                    lists.append(pos if t else [])
            slops.append(min_slop(lists))
        return values, scores, boost, tuple(slops)

    def total(self, scores, boost):
        t = 0.0
        for (_k, _f, _c, _col, coeff), s in zip(self.ops, scores):
            t = t + coeff * s
        return t * boost
