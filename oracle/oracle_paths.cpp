// oracle/oracle_paths.cpp -- CPU restatement of the webgraph's shortest-path search and of ApproxHarmonic.
// TEST INFRASTRUCTURE ONLY (see oracle_common.h).  Follows, by file:line in /root/reference:
//   crates/core/src/webgraph/shortest_path.rs:57-105     dijkstra_multi (binary heap, u8 costs, the max_dist cut-off
//                                                        that fires when a node with cost > max_dist is POPPED)
//   crates/core/src/webgraph/centrality/approx_harmonic.rs:40-88   ApproxHarmonic::build for a given sample
// The graph is handed over as the unique (from, to) links the search may follow, with dense node ranks (positions in
// ascending id order), which is what tests derive from the oracle's own staging (orc_hb_dense_*).
// Parity status: the reference holds no numeric golden for either function; ApproxHarmonic's own result is not
// deterministic (random sample; f32 terms accumulated in a DashMap from a rayon pool), so parity is on the distances
// (exact) and, for a fixed sample, on the sums within f32 accumulation error.
#include "oracle_common.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <functional>
#include <queue>
#include <vector>

namespace {
struct Csr { std::vector<uint64_t> ptr; std::vector<uint32_t> adj; };
static Csr build(uint32_t n, const uint32_t* from, const uint32_t* to, uint64_t m, bool reversed) {
  Csr c; c.ptr.assign((size_t)n + 1, 0); c.adj.resize(m);
  for (uint64_t e = 0; e < m; e++) c.ptr[(reversed ? to[e] : from[e]) + 1]++;
  for (uint32_t v = 0; v < n; v++) c.ptr[v + 1] += c.ptr[v];
  std::vector<uint64_t> pos(c.ptr.begin(), c.ptr.end() - 1);
  for (uint64_t e = 0; e < m; e++) { const uint32_t a = reversed ? to[e] : from[e], b = reversed ? from[e] : to[e]; c.adj[pos[a]++] = b; }
  return c;
}
// dijkstra_multi: `dist` must be filled with 255 ("not in the map")
static void dijkstra_multi(const Csr& g, const uint32_t* sources, uint32_t n_sources, int max_dist /* < 0: None */, uint8_t* dist) {
  typedef std::pair<uint8_t, uint32_t> St;
  std::priority_queue<St, std::vector<St>, std::greater<St>> q;   // BinaryHeap of Reverse((cost, node))
  for (uint32_t i = 0; i < n_sources; i++) {
    if (sources[i] == 0xFFFFFFFFu) continue;   // an id that is not a node reaches nothing (the device skips it too)
    q.push({0, sources[i]}); dist[sources[i]] = 0;
  }
  while (!q.empty()) {
    const St st = q.top(); q.pop();
    const uint8_t cost = st.first; const uint32_t v = st.second;
    if (cost > dist[v]) continue;
    if (max_dist >= 0 && cost > max_dist) return;
    for (uint64_t e = g.ptr[v]; e < g.ptr[v + 1]; e++) {
      const uint32_t w = g.adj[e];
      if ((int)cost + 1 < (int)dist[w]) { dist[w] = (uint8_t)(cost + 1); q.push({(uint8_t)(cost + 1), w}); }
    }
  }
}
}  // namespace

// one search per group: sources with group[i] == s start search s together.  dist_out [n_groups][n], 255 = not reached
ORC_API void orc_graph_distances(uint32_t n, const uint32_t* from, const uint32_t* to, uint64_t m, const uint32_t* sources,
                                 const uint32_t* group, uint32_t n_sources, uint32_t n_groups, int max_dist, int reversed, uint8_t* dist_out) {
  const Csr g = build(n, from, to, m, reversed != 0);
  memset(dist_out, 255, (size_t)n_groups * n);
  for (uint32_t s = 0; s < n_groups; s++) {
    std::vector<uint32_t> src;
    for (uint32_t i = 0; i < n_sources; i++) if (group[i] == s) src.push_back(sources[i]);
    if (!src.empty()) dijkstra_multi(g, src.data(), (uint32_t)src.size(), max_dist, dist_out + (size_t)s * n);
  }
}

// ApproxHarmonic::build for the sample `sources` (ranks), sources taken in the order given; out32 = the reference's f32
// accumulation in that order, out64 = the same f32 terms summed in f64 (what the device path computes); 0 = not reached
ORC_API void orc_approx_harmonic(uint32_t n, const uint32_t* from, const uint32_t* to, uint64_t m, const uint32_t* sources,
                                 uint32_t n_sources, int max_dist, uint64_t num_nodes, float* out32, double* out64) {
  const Csr g = build(n, from, to, m, false);
  const float nn = (float)num_nodes;
  const float norm = nn / ((float)n_sources * (nn - 1.0f));
  std::vector<uint8_t> dist(n);
  for (uint32_t v = 0; v < n; v++) { out32[v] = 0.0f; out64[v] = 0.0; }
  for (uint32_t i = 0; i < n_sources; i++) {
    std::fill(dist.begin(), dist.end(), (uint8_t)255);
    dijkstra_multi(g, sources + i, 1, max_dist, dist.data());
    for (uint32_t v = 0; v < n; v++) {
      if (dist[v] == 255 || dist[v] == 0) continue;
      const float term = (1.0f / (float)dist[v]) * norm;
      out32[v] += term; out64[v] += (double)term;
    }
  }
}

// ---------------------------------------------------------------- inbound similarity ---------
// bitvec_similarity.rs:24-185 + inbound_similarity.rs:26-119.  The graph comes as unique links over dense ranks (self-links
// included) plus the node ids; liked / disliked / candidates are ranks, 0xFFFFFFFF = the one id that is not a node.
namespace {
struct BitVecO {
  std::vector<u128> ranks; uint64_t bloom[16]; size_t ones = 0; double sqrt_len = 0;
  void build(std::vector<u128> v) {   // BitVec::new
    std::sort(v.begin(), v.end()); v.erase(std::unique(v.begin(), v.end()), v.end());
    memset(bloom, 0, sizeof(bloom)); ones = 0;
    for (u128 r : v) {               // VeryJankyBloomFilter::insert_u128 -> insert(item as u64)
      const uint64_t h = (uint64_t)r * 11400714819323198549ull;
      const size_t a = (size_t)(h % 16); const uint64_t b = h % 64;
      if (bloom[a] & (1ull << b)) continue;
      bloom[a] |= 1ull << b; ones++;
    }
    sqrt_len = std::sqrt((double)v.size());
    ranks.swap(v);
  }
  double sim(const BitVecO& o) const {   // BitVec::sim
    if (sqrt_len == 0.0 || o.sqrt_len == 0.0) return 0.0;
    const size_t mx = std::max(ones, o.ones);
    size_t inter = 0;
    for (int i = 0; i < 16; i++) inter += (size_t)__builtin_popcountll(bloom[i] & o.bloom[i]);
    if ((double)inter / (double)mx < 0.25) return 0.0;
    size_t i = 0, j = 0, c = 0;
    while (i < ranks.size() && j < o.ranks.size()) { if (ranks[i] == o.ranks[j]) { c++; i++; j++; } else if (ranks[i] < o.ranks[j]) i++; else j++; }
    return (double)c / (sqrt_len * o.sqrt_len);
  }
};
}  // namespace
ORC_API void orc_inbound_similarity(uint32_t n, const uint64_t* id_lo, const uint64_t* id_hi, const uint32_t* from, const uint32_t* to, uint64_t m,
                                    const uint32_t* liked, uint32_t n_liked, const uint32_t* disliked, uint32_t n_disliked,
                                    const uint32_t* cand, uint32_t n_cand, int normalized, double self_score, double* out) {
  const Csr in = build(n, from, to, m, true);   // ingoing: adjacency of `to`
  auto inbound = [&](uint32_t r) {
    BitVecO b; std::vector<u128> v;
    if (r != 0xFFFFFFFFu) for (uint64_t e = in.ptr[r]; e < in.ptr[r + 1]; e++) v.push_back(orc_make_u128(id_hi[in.adj[e]], id_lo[in.adj[e]]));
    b.build(std::move(v));
    return b;
  };
  std::vector<BitVecO> L(n_liked), D(n_disliked);
  for (uint32_t i = 0; i < n_liked; i++) L[i] = inbound(liked[i]);
  for (uint32_t i = 0; i < n_disliked; i++) D[i] = inbound(disliked[i]);
  for (uint32_t c = 0; c < n_cand; c++) {
    const BitVecO cb = inbound(cand[c]);
    double ls = 0.0, ds = 0.0;   // NodeScorer::sim compares NodeIDs: equal ranks = the same node (0xFFFFFFFF stands for ONE id that is not in the graph)
    for (uint32_t i = 0; i < n_liked; i++) ls += liked[i] == cand[c] ? self_score : L[i].sim(cb);
    for (uint32_t i = 0; i < n_disliked; i++) ds += disliked[i] == cand[c] ? self_score : D[i].sim(cb);
    double s = (double)n_disliked + (ls - ds);
    if (normalized) s = s / (double)std::max<uint32_t>(n_liked, 1);
    out[c] = std::max(s, 0.0);
  }
}
