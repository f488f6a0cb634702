// phrase_oracle_mt.cpp -- the phrase-query oracle of tests/phrase_oracle.py restated in C++ with a batch driver that runs
// one query per host thread (test and benchmark infrastructure: the CPU baseline and the parity reference at benchmark
// size).  tests/test_oracle_phrase_native.py pins it against the Python oracle, which is pinned on the reference's tests.
//
// Index: term t owns postings [term_off[t], term_off[t+1]) with ascending docs; posting p owns the absolute ascending
// positions [pos_off[p], pos_off[p+1]).  A query row holds term ids in offset order, 0xFFFFFFFF pads the end, 0xFFFFFFFE is
// a term the segment does not hold.  Scoring: count = PhraseScorer::compute_phrase_count, score = weight * (count / (count +
// cache[fieldnorm id])) in f32; scoring off: phrase_exists, score 1.  Top-k by (score desc, doc asc).
#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cstdlib>
#include <thread>
#include <vector>

namespace {

using V = std::vector<uint32_t>;
inline uint32_t adiff(uint32_t a, uint32_t b) { return a > b ? a - b : b - a; }

V intersection(const V& l, const V& r) {
  V out; size_t i = 0, j = 0;
  while (i < l.size() && j < r.size()) {
    if (l[i] < r[j]) i++; else if (l[i] == r[j]) { out.push_back(l[i]); i++; j++; } else j++;
  }
  return out;
}
uint32_t intersection_count(const V& l, const V& r) { return (uint32_t)intersection(l, r).size(); }
bool intersection_exists(const V& l, const V& r) { return !intersection(l, r).empty(); }

uint32_t count_with_slop(V& l, const V& r, uint32_t slop, bool update) {
  size_t i = 0, j = 0; uint32_t c = 0; V out;
  while (i < l.size() && j < r.size()) {
    const uint32_t lv = l[i], rv = r[j];
    if (adiff(lv, rv) <= slop) {
      while (i + 1 < l.size() && l[i + 1] <= rv) i++;
      out.push_back(rv); c++; i++; j++;
    } else if (lv < rv) i++; else j++;
  }
  if (update) l = out;
  return c;
}
bool exists_with_slop(const V& l, const V& r, uint32_t slop) {
  size_t i = 0, j = 0;
  while (i < l.size() && j < r.size()) {
    if (adiff(l[i], r[j]) <= slop) return true;
    if (l[i] < r[j]) i++; else j++;
  }
  return false;
}
uint32_t carrying(V& l, std::vector<uint8_t>& ls, const V& r, uint32_t max_slop, bool update) {
  if (l.empty() || r.empty()) { if (update) { l.clear(); ls.clear(); } return 0; }
  V pb; std::vector<uint8_t> sb;
  auto add = [&](uint32_t s, uint32_t v) {
    if (!update) return;
    if (!pb.empty() && pb.back() == v) sb.back() = std::min<uint8_t>(sb.back(), (uint8_t)s);
    else { pb.push_back(v); sb.push_back((uint8_t)s); }
  };
  size_t i = 0, j = 0; uint32_t count = 0;
  for (;;) {
    const uint32_t lv = l[i], rv = r[j], sso = i < ls.size() ? ls[i] : 0u;
    const uint32_t dist = sso + adiff(lv, rv);
    if (dist <= max_slop) {
      const bool lsm = lv < rv;
      const uint32_t larger = lsm ? rv : lv;
      const V& sp = lsm ? l : r; size_t si = lsm ? i : j;
      uint32_t ns = dist;
      add(ns, lsm ? lv : rv);
      while (si + 1 < sp.size()) { const uint32_t nv = sp[si + 1]; if (nv > larger) break; si++; ns = sso + adiff(nv, larger); add(ns, nv); }
      add(ns, larger);
      count++; i++; j++;
    } else if (lv < rv) i++; else j++;
    if (i >= l.size() || j >= r.size()) {
      if (i >= l.size()) {
        const uint32_t lv2 = l.back(), s2 = ls.empty() ? 0u : ls.back();
        for (size_t x = j; x < r.size(); x++) { const uint32_t s = adiff(lv2, r[x]) + s2; if (s <= max_slop) add(s, r[x]); }
      } else {
        const uint32_t rv2 = r.back();
        for (size_t x = i; x < l.size(); x++) { const uint32_t s = adiff(l[x], rv2) + (x < ls.size() ? ls[x] : 0u); if (s <= max_slop) add(s, l[x]); }
      }
      break;
    }
  }
  if (update) { l.swap(pb); ls.swap(sb); }
  return count;
}

uint32_t phrase_match(const std::vector<V>& lists, uint32_t slop, bool scoring) {
  const size_t n = lists.size();
  V left = lists[0]; std::vector<uint8_t> ls;
  for (size_t i = 1; i + 1 < n; i++) {
    if (slop > 0) { if (n > 2) carrying(left, ls, lists[i], slop, true); else count_with_slop(left, lists[i], slop, true); }
    else left = intersection(left, lists[i]);
    if (left.empty()) return 0;
  }
  const V& right = lists[n - 1];
  if (scoring) {
    if (slop > 0) return n > 2 ? carrying(left, ls, right, slop, false) : count_with_slop(left, right, slop, false);
    return intersection_count(left, right);
  }
  return (slop > 0 ? exists_with_slop(left, right, slop) : intersection_exists(left, right)) ? 1u : 0u;
}

struct Hit { float s; uint32_t d; };

}  // namespace

extern "C" int phrase_oracle_batch(const uint32_t* docs, const uint64_t* term_off, uint32_t n_terms, const uint32_t* positions,
                                   const uint64_t* pos_off, const uint8_t* fieldnorm_ids, const float* cache, uint32_t nq, uint32_t nt,
                                   const uint32_t* rows, const uint32_t* offsets, const uint32_t* slops, const float* weights, int scoring,
                                   uint32_t k, uint32_t* out_docs, float* out_scores, uint32_t* out_n, int threads) {
  std::atomic<uint32_t> next(0);
  std::atomic<int> bad(0);
  auto work = [&]() {
    for (uint32_t q; (q = next.fetch_add(1)) < nq;) {
      out_n[q] = 0;
      std::vector<std::pair<uint32_t, uint32_t>> terms;   // (term, shift) in offset order
      bool absent = false; uint32_t max_off = 0;
      for (uint32_t j = 0; j < nt; j++) {
        const uint32_t t = rows[(size_t)q * nt + j];
        if (t == 0xFFFFFFFFu) break;
        if (t == 0xFFFFFFFEu) absent = true;
        else if (t >= n_terms) { bad = 1; absent = true; }
        max_off = std::max(max_off, offsets[(size_t)q * nt + j]);
        terms.push_back({t, offsets[(size_t)q * nt + j]});
      }
      if (absent || terms.size() < 2) continue;
      for (auto& p : terms) p.second = max_off - p.second;
      std::stable_sort(terms.begin(), terms.end(), [&](const std::pair<uint32_t, uint32_t>& a, const std::pair<uint32_t, uint32_t>& b) {
        return term_off[a.first + 1] - term_off[a.first] < term_off[b.first + 1] - term_off[b.first]; });
      std::vector<uint64_t> cur(terms.size());
      for (size_t i = 0; i < terms.size(); i++) cur[i] = term_off[terms[i].first];
      std::vector<Hit> hits;
      std::vector<V> lists(terms.size());
      const uint64_t a_end = term_off[terms[0].first + 1];
      for (uint64_t pa = cur[0]; pa < a_end; pa++) {
        const uint32_t doc = docs[pa];
        bool all = true;
        std::vector<uint64_t> at(terms.size()); at[0] = pa;
        for (size_t i = 1; i < terms.size() && all; i++) {
          const uint64_t e = term_off[terms[i].first + 1];
          cur[i] = std::lower_bound(docs + cur[i], docs + e, doc) - docs;   // seek
          all = cur[i] < e && docs[cur[i]] == doc; at[i] = cur[i];
        }
        if (!all) continue;
        for (size_t i = 0; i < terms.size(); i++) {
          lists[i].assign(positions + pos_off[at[i]], positions + pos_off[at[i] + 1]);
          for (auto& x : lists[i]) x += terms[i].second;
        }
        const uint32_t c = phrase_match(lists, slops[q], scoring != 0);
        if (!c) continue;
        float s = 1.0f;
        if (scoring) { const volatile float tf = (float)c; const volatile float f = tf / (tf + cache[fieldnorm_ids[doc]]); s = weights[q] * f; }
        hits.push_back({s, doc});
      }
      const size_t m = std::min<size_t>(k, hits.size());
      std::partial_sort(hits.begin(), hits.begin() + m, hits.end(), [](const Hit& a, const Hit& b) { return a.s > b.s || (a.s == b.s && a.d < b.d); });
      for (size_t i = 0; i < m; i++) { out_docs[(size_t)q * k + i] = hits[i].d; out_scores[(size_t)q * k + i] = hits[i].s; }
      out_n[q] = (uint32_t)m;
    }
  };
  std::vector<std::thread> pool;
  for (int i = 0; i < std::max(1, threads); i++) pool.emplace_back(work);
  for (auto& th : pool) th.join();
  return bad ? 1 : 0;
}
