// The canonical-order restatement of Betweenness::calculate (crates/core/src/webgraph/centrality/betweenness.rs:29-146),
// threaded over sources: the bit-exact reference of the device betweenness and the CPU baseline of
// tools/betweenness_bench.py.  Test infrastructure, compiled into a temporary directory by tests/betweenness_oracle.py.
//
// Per source s (i32 sigma wrapping like the reference's release build, f64 without contraction):
//   BFS over the out-links; sigma[w] += sigma[v] over every v -> w with dist[w] == dist[v] + 1;
//   in reverse visit order, delta[v] = delta[v] + (sigma[v] as f64 / sigma[w] as f64) * (1.0 + delta[w]) over v's
//   successors w ascending in node id (the canonical order; the reference's follows the store's link order);
//   centrality[w] += delta[w] for every reached w != s, sources in the given order.
#include <stdint.h>

#include <algorithm>
#include <thread>
#include <vector>

namespace {

struct Csr {
  std::vector<uint32_t> ptr, dst;
};

struct Search {
  std::vector<int32_t> dist;
  std::vector<uint32_t> sigma;
  std::vector<uint32_t> order;
  explicit Search(uint32_t n) : dist(n, -1), sigma(n, 0) { order.reserve(n); }

  // delta (dense, 0.0 where unreached and at s) of one source; returns the deepest distance
  int32_t run(const Csr& g, uint32_t s, double* delta) {
    std::fill(delta, delta + dist.size(), 0.0);
    order.clear();
    dist[s] = 0; sigma[s] = 1; order.push_back(s);
    for (size_t h = 0; h < order.size(); h++) {
      const uint32_t v = order[h];
      for (uint32_t e = g.ptr[v]; e < g.ptr[v + 1]; e++) {
        const uint32_t w = g.dst[e];
        if (dist[w] < 0) { dist[w] = dist[v] + 1; order.push_back(w); }
        if (dist[w] == dist[v] + 1) sigma[w] += sigma[v];   // u32 addition wraps exactly like the i32 one
      }
    }
    for (size_t h = order.size(); h-- > 0;) {
      const uint32_t v = order[h];
      double d = 0.0;
      for (uint32_t e = g.ptr[v]; e < g.ptr[v + 1]; e++) {
        const uint32_t w = g.dst[e];
        if (dist[w] == dist[v] + 1) d = d + ((double)(int32_t)sigma[v] / (double)(int32_t)sigma[w]) * (1.0 + delta[w]);
      }
      delta[v] = d;
    }
    const int32_t deepest = dist[order.back()];
    delta[s] = 0.0;   // not added: w != s
    for (uint32_t v : order) { dist[v] = -1; sigma[v] = 0; }
    return deepest;
  }
};

}  // namespace

extern "C" {

// n nodes, m links (from_rank -> to_rank, self-loops and repeats allowed: both are dropped), n_sources distinct ranks.
// Adds the sources' dependencies, in source order, to centrality [n] (not normalised: a caller may continue with further
// sources), marks reached [n] (the key set: sources and every node a source reaches) and raises *max_dist.
// Returns 0, or -1 for a source rank >= n.
int bc_oracle(uint32_t n, const uint32_t* from_rank, const uint32_t* to_rank, uint64_t m, const uint32_t* sources, uint32_t n_sources,
              int threads, double* centrality, uint8_t* reached, int32_t* max_dist) {
  for (uint32_t i = 0; i < n_sources; i++) if (sources[i] >= n) return -1;
  Csr g;
  {
    std::vector<uint64_t> keys;
    keys.reserve(m);
    for (uint64_t i = 0; i < m; i++) if (from_rank[i] != to_rank[i]) keys.push_back((uint64_t)from_rank[i] << 32 | to_rank[i]);
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    g.ptr.assign(n + 1, 0); g.dst.resize(keys.size());
    for (size_t i = 0; i < keys.size(); i++) { g.ptr[(keys[i] >> 32) + 1]++; g.dst[i] = (uint32_t)keys[i]; }
    for (uint32_t v = 0; v < n; v++) g.ptr[v + 1] += g.ptr[v];
  }
  if (threads < 1) threads = 1;
  // rounds of `round` sources: each thread fills the dense deltas of its sources, then the rounds' deltas are added per
  // node in source order (threads own node ranges); adding the 0.0 of an unreached node leaves the sum unchanged
  const uint32_t round = (uint32_t)threads * 4;
  std::vector<double> delta((size_t)round * n);
  std::vector<int32_t> deep(round);
  std::vector<Search> searches;
  for (int t = 0; t < threads; t++) searches.emplace_back(n);
  for (uint32_t base = 0; base < n_sources; base += round) {
    const uint32_t k = std::min(round, n_sources - base);
    std::vector<std::thread> pool;
    for (int t = 0; t < threads; t++)
      pool.emplace_back([&, t] {
        for (uint32_t j = t; j < k; j += threads) deep[j] = searches[t].run(g, sources[base + j], delta.data() + (size_t)j * n);
      });
    for (auto& th : pool) th.join();
    pool.clear();
    for (int t = 0; t < threads; t++)
      pool.emplace_back([&, t] {
        const uint32_t a = (uint32_t)((uint64_t)n * t / threads), b = (uint32_t)((uint64_t)n * (t + 1) / threads);
        for (uint32_t j = 0; j < k; j++) {
          const double* d = delta.data() + (size_t)j * n;
          for (uint32_t v = a; v < b; v++) centrality[v] = centrality[v] + d[v];
        }
      });
    for (auto& th : pool) th.join();
    for (uint32_t j = 0; j < k; j++) *max_dist = std::max(*max_dist, deep[j]);
  }
  // the key set: BFS reachability from every source (a node with 0.0 still has an entry)
  {
    std::vector<uint32_t> stack;
    for (uint32_t i = 0; i < n_sources; i++) {
      const uint32_t s = sources[i];
      if (reached[s]) continue;   // everything a marked node reaches is marked (in this call or an earlier one)
      reached[s] = 1; stack.push_back(s);
      while (!stack.empty()) {
        const uint32_t v = stack.back(); stack.pop_back();
        for (uint32_t e = g.ptr[v]; e < g.ptr[v + 1]; e++) if (!reached[g.dst[e]]) { reached[g.dst[e]] = 1; stack.push_back(g.dst[e]); }
      }
    }
  }
  return 0;
}

}  // extern "C"
