"""Host-side mirror of Stract's recall-stage collector (crates/core/src/collector/top_docs.rs), the step that sits right
behind the GPU's top-k by `total`.

  CollectorConfig        crates/core/src/config/{mod.rs, defaults.rs:21-40}
  Hashes / BucketCount / BucketCollector   top_docs.rs:213-373 (site / url / url-without-tld / title buckets, simhash table)
  simhash::Table         crates/core/src/simhash.rs:69-135 (a hash within Hamming distance 3 of an inserted one)

The collector is sequential by construction (every pick changes the penalties of the remaining documents), so it stays on
the host -- like the reference's, which runs it once per segment at harvest time over at most `max_docs_considered`
documents.  What the GPU contributes is the candidate list: `harvest_top_k` feeds the collector the top-K documents by
`total` and proves K was enough (see there).

Order: documents pop by `f64::total_cmp` on the adjusted score, as `ScoredDoc::cmp` orders them (top_docs.rs:229-233), so
-0.0 sits below +0.0, -inf below every number and a NaN ranks by its sign bit (a positive NaN above +inf, a negative one below
-inf).  The reference's `update_best_doc` compares the re-adjusted score with `==`, which never holds for a NaN, so a NaN best
document would loop there forever; this mirror compares the two scores' bits instead and so ranks a NaN by its bits and
terminates.  The device's top-k hands every NaN total over as the negative NaN 0xFFF8000000000000 (DESIGN §5), which this
order puts last.

Tie note: the reference keeps the documents in a `min_max_heap::MinMaxHeap`; which of two documents with EQUAL adjusted
score pops first is a property of that crate (not part of the reference tree).  This mirror pops the earlier-inserted one.
"""
import heapq
import struct

import numpy as np


def total_cmp_key(x):
    """An int that orders f64 values as `f64::total_cmp` does (core::f64::total_cmp: flip the magnitude bits of negatives)."""
    b = struct.unpack("<q", struct.pack("<d", float(x)))[0]
    return b ^ 0x7FFFFFFFFFFFFFFF if b < 0 else b


class CollectorConfig:
    """config/defaults.rs:21-40."""

    def __init__(self, site_penalty=0.1, title_penalty=1.0, url_penalty=20.0, url_without_tld_penalty=1.0, max_docs_considered=250_000):
        self.site_penalty, self.title_penalty, self.url_penalty = site_penalty, title_penalty, url_penalty
        self.url_without_tld_penalty, self.max_docs_considered = url_without_tld_penalty, max_docs_considered


class Hashes:
    __slots__ = ("site", "title", "url", "url_without_tld", "simhash")

    def __init__(self, site, title, url, url_without_tld, simhash):
        self.site, self.title, self.url, self.url_without_tld, self.simhash = int(site), int(title), int(url), int(url_without_tld), int(simhash)


class SimhashTable:
    """simhash::Table: `contains` is true iff an inserted hash lies within Hamming distance K = 3 (the four 16-bit blocks are
    the pigeonhole index that makes the lookup fast in the reference; the predicate is exactly this)."""
    K = 3

    def __init__(self):
        self._h = []

    def insert(self, h):
        self._h.append(int(h))

    def contains(self, h):
        h = int(h)
        return any(bin(h ^ x).count("1") <= self.K for x in self._h)


class BucketCollector:
    """top_docs.rs:289-373.  Documents are (score, hashes, payload); `into_sorted_vec` returns the payloads."""

    def __init__(self, top_n, config=None):
        assert top_n > 0
        self.top_n = top_n
        self.config = config or CollectorConfig()
        self.buckets = {}
        self._heap = []   # (-total_cmp_key(adjusted score), insertion index, adjusted score, score, hashes, payload)
        self._seq = 0

    def _adjusted(self, score, h):
        b, c = self.buckets, self.config
        # the four hash spaces share one HashMap<Prehashed, usize> in the reference (top_docs.rs:247-249)
        adjuster = 1.0 / (1.0 + b.get(h.site, 0) * c.site_penalty + b.get(h.url, 0) * c.url_penalty
                          + b.get(h.url_without_tld, 0) * c.url_without_tld_penalty + b.get(h.title, 0) * c.title_penalty)
        return score * adjuster

    def insert(self, score, hashes, payload=None):
        adj = self._adjusted(score, hashes)
        heapq.heappush(self._heap, (-total_cmp_key(adj), self._seq, adj, float(score), hashes, payload))
        self._seq += 1

    def _update_counts(self, h):
        for key in (h.site, h.url, h.url_without_tld, h.title):
            self.buckets[key] = self.buckets.get(key, 0) + 1

    def _update_best_doc(self):
        if len(self._heap) <= 1:
            return
        while self._heap:
            neg, seq, _adj, score, h, payload = self._heap[0]
            new = self._adjusted(score, h)
            if total_cmp_key(new) == -neg:   # the same bits (the reference's `==` would never end on a NaN)
                break
            heapq.heapreplace(self._heap, (-total_cmp_key(new), seq, new, score, h, payload))

    def into_sorted_vec(self, de_rank_similar=True, with_adjusted=False):
        res, dups, table = [], [], SimhashTable()
        while self._heap:
            _neg, _seq, adj, score, h, payload = heapq.heappop(self._heap)
            if h.simhash != 0 and de_rank_similar:
                if table.contains(h.simhash):
                    dups.append((payload, adj))
                    continue
                table.insert(h.simhash)
            if de_rank_similar:
                self._update_counts(h)
                self._update_best_doc()
            res.append((payload, adj))
            if len(res) == self.top_n:
                break
        res.extend(dups[:max(self.top_n - len(res), 0)])
        return res if with_adjusted else [p for p, _ in res]


def harvest_top_k(top_n, search, hashes_of, config=None, k0=None, k_max=4096):
    """TopSegmentCollector::harvest over a GPU candidate list.

    `search(K)` -> (docs, totals) = the top-K documents by (total desc, doc asc), e.g. one row of
    SignalComputer.top_docs_batch; `hashes_of(doc)` -> Hashes (the SiteHash / TitleHash / UrlHash / UrlWithoutTldHash /
    SimHash columns the reference reads at collect time, top_docs.rs:185-211).

    The reference inserts EVERY collected document; penalties only shrink positive scores, so a document outside the top-K
    can never beat a pick whose adjusted score is >= the K-th total.  The harvest over the top-K is therefore identical to
    the reference's as soon as either all candidates fit in K or every pick's adjusted score is >= the smallest total of the
    candidate list; otherwise K is doubled.  Returns ([(doc, total)], K used, proven) -- proven is False only when k_max was
    reached without a proof (the caller should widen the search)."""
    K = k0 or min(max(4 * top_n, 64), k_max)
    while True:
        docs, totals = search(K)
        bc = BucketCollector(top_n, config)
        for d, t in zip(docs, totals):
            bc.insert(float(t), hashes_of(int(d)), (int(d), float(t)))
        picks = bc.into_sorted_vec(True, with_adjusted=True)
        exhausted = len(docs) < K
        floor = float(totals[-1]) if len(totals) else 0.0
        proven = exhausted or (len(picks) == top_n and floor >= 0.0 and all(adj >= floor for _, adj in picks))
        if proven or K >= k_max:
            return [p for p, _ in picks], K, proven
        K = min(2 * K, k_max)
