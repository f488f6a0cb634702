// graph_betweenness.cu -- Brandes' betweenness centrality over the resident CSR, up to 64 sources per batch.
//
// Reference: Betweenness::calculate   crates/core/src/webgraph/centrality/betweenness.rs:29-146
//   per source s: BFS over the forward links counting shortest paths (sigma, an i32 that wraps), then the dependencies
//   delta[v] = delta[v] + (sigma[v] as f64 / sigma[w] as f64) * (1.0 + delta[w]) in reverse visit order;
//   centrality[w] += delta[w] for w != s; finally centrality / (n * (n - 1.0)), n = number of sources.
//
// Two orders the reference leaves to a hash set and to the store are pinned here (DESIGN §2 "Betweenness centrality"):
//   - centrality[w] sums the per-source delta[w] in the caller's source order (batches in order, bit b = source base + b);
//   - delta[v] sums over v's successors w on the shortest-path DAG in ascending node id of w.
//
// Layout of one batch of W sources (W = 64 unless the device is short of memory), node-major with the sources contiguous:
//   dist [N][W] u8 (255 = not reached), sigma [N][W] u32 (i32 wrapping arithmetic), delta [N][W] f64.
// Forward: the level loop of the bit-parallel search (graph_bfs.cu: seed, pull, commit); between the pull and the commit,
// k_bc_sigma adds, for every row discovered at this level, sigma[u][b] of the in-neighbours u on the previous level.
// Backward: level by level from the deepest, one warp per row, lane b (and b + 32) owns source b and walks the row's
// out-edges in ascending node id -- no floating-point atomics, so the result does not depend on scheduling.
#include "graph.cuh"

#ifndef SB200_EMU
#include <cub/cub.cuh>
#endif
#include <algorithm>
#include <vector>

namespace sb200 {

// source-major adjacency ordered by (source row, destination rank): key = src << 32 | rank(dst) for every kept edge
__global__ void k_bc_out_keys(uint64_t E, uint64_t N, const uint32_t* __restrict__ row_ptr, const uint32_t* __restrict__ col,
                              const uint32_t* __restrict__ perm, uint64_t* keys) {
  const uint64_t e = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (e >= E) return;
  uint64_t a = 0, b = N;   // the destination row of in-edge e: the last row starting at or before e
  while (b - a > 1) {
    const uint64_t m = (a + b) >> 1;
    if (row_ptr[m] <= e) a = m; else b = m;
  }
  keys[e] = ((uint64_t)col[e] << 32) | perm[a];
}
__global__ void k_bc_out_dst(const uint64_t* __restrict__ keys, uint64_t E, const uint32_t* __restrict__ inv, uint32_t* out_dst) {
  const uint64_t e = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (e < E) out_dst[e] = inv[(uint32_t)keys[e]];
}
__global__ void k_bc_seed(const uint32_t* __restrict__ seed_rank, const uint32_t* __restrict__ seed_bit, uint32_t n,
                          const uint32_t* __restrict__ inv, uint32_t W, uint8_t* dist, uint32_t* sigma) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t o = (uint64_t)inv[seed_rank[i]] * W + seed_bit[i];
  dist[o] = 0;
  sigma[o] = 1;
}
// forward, between the pull and the commit of `level`: one warp per work item of a long row (<= CHUNK_EDGES in-edges,
// partial sums combined with integer atomics, which are order-free) or per short row.  For every search b that reaches
// the row for the first time, sigma[row][b] = sum of sigma[u][b] over the in-neighbours u on the frontier of b.
__global__ void __launch_bounds__(256) k_bc_sigma(uint64_t n_items, const uint32_t* __restrict__ item_row, const uint32_t* __restrict__ item_start,
    uint32_t warp_row_begin, uint64_t quad_row_begin, uint64_t n_quad, const uint32_t* __restrict__ row_ptr, const uint32_t* __restrict__ col,
    const unsigned long long* __restrict__ frontier, const unsigned long long* __restrict__ next, const unsigned long long* __restrict__ visited,
    uint32_t W, uint32_t level, uint32_t* sigma, uint8_t* dist) {
  const uint64_t unit = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  if (unit >= n_items + n_quad) return;
  const uint32_t lane = threadIdx.x & 31;
  uint32_t row, e0, e1;
  bool whole = true, first = true;
  if (unit < n_items) {
    row = item_row[unit];
    const uint32_t c = (uint32_t)unit - item_start[row - warp_row_begin];
    e0 = row_ptr[row] + c * (uint32_t)CHUNK_EDGES; e1 = min(e0 + (uint32_t)CHUNK_EDGES, row_ptr[row + 1]);
    whole = false; first = c == 0;
  } else {
    row = (uint32_t)(quad_row_begin + (unit - n_items));
    e0 = row_ptr[row]; e1 = row_ptr[row + 1];
  }
  const unsigned long long nb = next[row] & ~visited[row];
  if (!nb) return;
  const bool hi = lane + 32 < W;
  uint32_t s0 = 0, s1 = 0;
  for (uint32_t base = e0; base < e1; base += 32) {
    const uint32_t e = base + lane;
    uint32_t u = 0;
    unsigned long long m = 0;
    if (e < e1) { u = col[e]; m = frontier[u] & nb; }
    unsigned bal = __ballot_sync(0xffffffffu, m != 0);
    while (bal) {
      const int j = __ffs(bal) - 1;
      bal &= bal - 1;
      const uint64_t ou = (uint64_t)__shfl_sync(0xffffffffu, u, j) * W;
      const unsigned long long mj = __shfl_sync(0xffffffffu, m, j);
      if ((mj >> lane) & 1) s0 += sigma[ou + lane];
      if (hi && ((mj >> (lane + 32)) & 1)) s1 += sigma[ou + lane + 32];
    }
  }
  const bool b0 = (nb >> lane) & 1, b1 = hi && ((nb >> (lane + 32)) & 1);
  uint32_t* sv = sigma + (uint64_t)row * W;
  if (whole) {
    if (b0) sv[lane] = s0;
    if (b1) sv[lane + 32] = s1;
  } else {
    if (b0 && s0) atomicAdd(sv + lane, s0);
    if (b1 && s1) atomicAdd(sv + lane + 32, s1);
  }
  if (first) {
    uint8_t* dv = dist + (uint64_t)row * W;
    if (b0) dv[lane] = (uint8_t)level;
    if (b1) dv[lane + 32] = (uint8_t)level;
  }
}
// backward, level `level` (>= 1): one warp per row v.  Lane b with dist[v][b] == level sums over v's out-edges in
// ascending node id, exactly as the reference's expression reads, the successors w with dist[w][b] == level + 1.
__global__ void __launch_bounds__(256) k_bc_delta(uint64_t N, const uint32_t* __restrict__ out_ptr, const uint32_t* __restrict__ out_dst,
    const uint8_t* __restrict__ dist, const uint32_t* __restrict__ sigma, double* delta, uint32_t W, uint32_t level) {
  const uint64_t v = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  if (v >= N) return;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t e0 = out_ptr[v], e1 = out_ptr[v + 1];
  if (e0 == e1) return;   // a sink keeps delta 0
  const uint64_t o = v * W;
  const bool a0 = lane < W && dist[o + lane] == level, a1 = lane + 32 < W && dist[o + lane + 32] == level;
  if (!__any_sync(0xffffffffu, a0 || a1)) return;
  const uint8_t nxt = (uint8_t)(level + 1);
  const double sv0 = a0 ? (double)(int32_t)sigma[o + lane] : 0.0, sv1 = a1 ? (double)(int32_t)sigma[o + lane + 32] : 0.0;
  double d0 = 0.0, d1 = 0.0;
  for (uint32_t base = e0; base < e1; base += 32) {
    const uint32_t wl = base + lane < e1 ? out_dst[base + lane] : 0;
    const uint32_t cnt = min(32u, e1 - base);
    for (uint32_t j = 0; j < cnt; j++) {
      const uint64_t ow = (uint64_t)__shfl_sync(0xffffffffu, wl, j) * W;
      if (a0 && dist[ow + lane] == nxt) d0 = d0 + (sv0 / (double)(int32_t)sigma[ow + lane]) * (1.0 + delta[ow + lane]);
      if (a1 && dist[ow + lane + 32] == nxt) d1 = d1 + (sv1 / (double)(int32_t)sigma[ow + lane + 32]) * (1.0 + delta[ow + lane + 32]);
    }
  }
  if (a0) delta[o + lane] = d0;
  if (a1) delta[o + lane + 32] = d1;
}
// after a batch: cent[v] += delta[v][b] for b in batch (= source) order over the searches that reached v, the source's own
// search excepted; every reached row is marked for the output
__global__ void __launch_bounds__(256) k_bc_accum(uint64_t N, const unsigned long long* __restrict__ visited, const uint8_t* __restrict__ dist,
    const double* __restrict__ delta, uint32_t W, double* cent, uint8_t* reached) {
  const uint64_t v = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  if (v >= N) return;
  const unsigned long long m = visited[v];
  if (!m) return;
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t o = v * W;
  const bool k0 = ((m >> lane) & 1) && dist[o + lane] != 0;
  const bool k1 = lane + 32 < W && ((m >> (lane + 32)) & 1) && dist[o + lane + 32] != 0;
  const double x0 = k0 ? delta[o + lane] : 0.0, x1 = k1 ? delta[o + lane + 32] : 0.0;
  const unsigned m0 = __ballot_sync(0xffffffffu, k0), m1 = __ballot_sync(0xffffffffu, k1);
  double c = cent[v];
  for (int b = 0; b < 32; b++) {
    const double y = __shfl_sync(0xffffffffu, x0, b);
    if ((m0 >> b) & 1) c = c + y;
  }
  for (int b = 0; b < 32; b++) {
    const double y = __shfl_sync(0xffffffffu, x1, b);
    if ((m1 >> b) & 1) c = c + y;
  }
  if (lane == 0) { cent[v] = c; reached[v] = 1; }
}
// rank order: the reached rows and their normalised centrality
__global__ void k_bc_flags(const uint32_t* __restrict__ inv, const double* __restrict__ cent, const uint8_t* __restrict__ reached, uint64_t N,
                           double norm, uint32_t* flag, double* val) {
  const uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (r >= N) return;
  const uint32_t v = inv[r];
  flag[r] = reached[v];
  val[r] = cent[v] / norm;
}

struct BcBatch {
  DevBuf<uint8_t> dist;
  DevBuf<uint32_t> sigma;
  DevBuf<double> delta;
  // the widest batch (64, 32, ... sources) whose per-node state fits: W * 13 bytes per node
  int alloc(uint64_t N, uint32_t& W) {
    for (W = 64; W >= 1; W >>= 1) {
      if (dist.alloc(N * W) == SB200_OK && sigma.alloc(N * W) == SB200_OK && delta.alloc(N * W) == SB200_OK) return SB200_OK;
      dist.release(); sigma.release(); delta.release();
    }
    return SB200_ENOMEM;
  }
};

}  // namespace sb200
using namespace sb200;

extern "C" {

int sb200_betweenness(sb200_graph* g, const uint64_t* src_lo, const uint64_t* src_hi, uint32_t n_sources, uint64_t* id_lo, uint64_t* id_hi,
                      double* centrality, uint64_t cap, uint64_t* len, uint32_t* max_dist) {
  if (!g) SB_FAIL(SB200_EINVAL, "NULL graph handle");
  SB_CUDA(cudaSetDevice(g->device));
  if (!len || !max_dist || (n_sources && (!src_lo || !src_hi))) SB_FAIL(SB200_EINVAL, "NULL argument");
  const uint64_t N = g->N;
  if (cap < N) SB_FAIL(SB200_EINVAL, "cap %llu < %llu nodes", (unsigned long long)cap, (unsigned long long)N);
  if (N && (!id_lo || !id_hi || !centrality)) SB_FAIL(SB200_EINVAL, "NULL output");
  *len = 0; *max_dist = 0;
  cudaStream_t s = g->stream;
  PoolScope scope(s);
  BfsState st;
  std::vector<uint32_t> ranks;
  SB_TRY(bfs_prepare(g, st, src_lo, src_hi, n_sources, ranks));
  {
    std::vector<uint8_t> seen(N, 0);
    for (uint32_t i = 0; i < n_sources; i++) {
      if (ranks[i] == 0xFFFFFFFFu) SB_FAIL(SB200_EINVAL, "source %u is not a node of the graph", i);
      if (seen[ranks[i]]++) SB_FAIL(SB200_EINVAL, "source %u repeats an earlier source", i);
    }
  }
  if (!n_sources) return SB200_OK;
  const int TPB = 256;
  const uint64_t E = g->E_kept;

  // out-rows ascending in node id (the canonical order of the dependency sums)
  DevBuf<uint32_t> out_ptr, out_dst;
  SB_TRY(out_ptr.alloc(N + 1));
  SB_CUDA(cudaMemsetAsync(out_ptr.p, 0, (N + 1) * 4, s));
  if (E) {
    DevBuf<uint64_t> ka, kb;
    SB_TRY(ka.alloc(E)); SB_TRY(kb.alloc(E)); SB_TRY(out_dst.alloc(E));
    SB_LAUNCH(k_bc_out_keys, div_up(E, TPB), TPB, 0, s, E, N, g->row_ptr.p, g->col.p, g->perm.p, ka.p);
    SB_CHECK_LAUNCH();
    int nbits = 1;
    while (nbits < 32 && (1ull << nbits) < N) nbits++;
    cub::DoubleBuffer<uint64_t> dk(ka.p, kb.p);
    size_t need = 0;
    DevBuf<uint8_t> tmp;   // scratch of this call: the handle keeps nothing
    SB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, need, dk, (int64_t)E, 0, 32 + nbits, s));
    SB_TRY(tmp.alloc(need + 256));
    SB_CUDA(cub::DeviceRadixSort::SortKeys(tmp.p, need, dk, (int64_t)E, 0, 32 + nbits, s));
    g_launches.fetch_add(8, std::memory_order_relaxed);
    SB_LAUNCH(k_bc_out_dst, div_up(E, TPB), TPB, 0, s, dk.Current(), E, g->inv.p, out_dst.p);
    SB_CHECK_LAUNCH();
    SB_LAUNCH(k_offsets_from_sorted, div_up(E + 1, TPB), TPB, 0, s, dk.Current(), E, N, out_ptr.p);
    SB_CHECK_LAUNCH();
    SB_CUDA(cudaStreamSynchronize(s));   // ka / kb go out of scope
  }

  BcBatch bt;
  uint32_t W = 64;
  SB_TRY(bt.alloc(N, W));
  DevBuf<double> cent; DevBuf<uint8_t> reached;
  SB_TRY(cent.alloc(N)); SB_TRY(reached.alloc(N));
  SB_CUDA(cudaMemsetAsync(cent.p, 0, N * 8, s)); SB_CUDA(cudaMemsetAsync(reached.p, 0, N, s));
  SB_TRY(st.seed_rank.alloc(W)); SB_TRY(st.seed_bit.alloc(W));
  const uint64_t nq = g->quad_row_end - g->quad_row_begin, units = g->n_items + nq;
  uint32_t deepest = 0;
  for (uint32_t base = 0; base < n_sources; base += W) {
    const uint32_t nb = std::min(n_sources - base, W);
    std::vector<uint32_t> sr(ranks.begin() + base, ranks.begin() + base + nb), sbit(nb);
    for (uint32_t i = 0; i < nb; i++) sbit[i] = i;
    SB_CUDA(cudaMemcpyAsync(st.seed_rank.p, sr.data(), nb * 4, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(st.seed_bit.p, sbit.data(), nb * 4, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemsetAsync(st.frontier.p, 0, N * 8, s)); SB_CUDA(cudaMemsetAsync(st.next.p, 0, N * 8, s));
    SB_CUDA(cudaMemsetAsync(st.visited.p, 0, N * 8, s));
    SB_CUDA(cudaMemsetAsync(bt.dist.p, 0xFF, N * W, s)); SB_CUDA(cudaMemsetAsync(bt.sigma.p, 0, N * W * 4, s));
    SB_CUDA(cudaMemsetAsync(bt.delta.p, 0, N * W * 8, s));
    SB_LAUNCH(k_bfs_seed, div_up(nb, TPB), TPB, 0, s, st.seed_rank.p, st.seed_bit.p, nb, g->inv.p, st.frontier.p, st.visited.p);
    SB_CHECK_LAUNCH();
    SB_LAUNCH(k_bc_seed, div_up(nb, TPB), TPB, 0, s, st.seed_rank.p, st.seed_bit.p, nb, g->inv.p, W, bt.dist.p, bt.sigma.p);
    SB_CHECK_LAUNCH();
    uint32_t depth = 0;
    for (uint32_t level = 1;; level++) {
      if (g->n_items) {
        SB_LAUNCH(k_bfs_pull_items, div_up(g->n_items * 32, TPB), TPB, 0, s, g->n_items, g->item_row.p, g->item_start.p, (uint32_t)g->warp_row_begin,
                  g->row_ptr.p, g->col.p, st.frontier.p, st.next.p);
        SB_CHECK_LAUNCH();
      }
      if (nq) {
        SB_LAUNCH(k_bfs_pull_rows, div_up(nq, TPB), TPB, 0, s, g->quad_row_begin, g->quad_row_end, g->row_ptr.p, g->col.p, st.frontier.p, st.next.p);
        SB_CHECK_LAUNCH();
      }
      if (units) {
        SB_LAUNCH(k_bc_sigma, div_up(units * 32, TPB), TPB, 0, s, g->n_items, g->item_row.p, g->item_start.p, (uint32_t)g->warp_row_begin,
                  g->quad_row_begin, nq, g->row_ptr.p, g->col.p, st.frontier.p, st.next.p, st.visited.p, W, level, bt.sigma.p, bt.dist.p);
        SB_CHECK_LAUNCH();
      }
      SB_CUDA(cudaMemsetAsync(st.any.p, 0, 8, s));
      SB_LAUNCH(k_bfs_commit, div_up(N, TPB), TPB, 0, s, N, g->perm.p, st.next.p, st.visited.p, st.frontier.p, level, nullptr, 0u, nullptr, 0.0,
                st.any.p);
      SB_CHECK_LAUNCH();
      unsigned long long any = 0;
      SB_CUDA(cudaMemcpyAsync(&any, st.any.p, 8, cudaMemcpyDeviceToHost, s));
      SB_CUDA(cudaStreamSynchronize(s));
      if (!any) break;
      if (level > 254) SB_FAIL(SB200_ERANGE, "source %u reaches a node at distance 255 (distances are u8)", base);
      depth = level;
    }
    deepest = std::max(deepest, depth);
    for (uint32_t level = depth; level-- > 1;) {
      SB_LAUNCH(k_bc_delta, div_up(N * 32, TPB), TPB, 0, s, N, out_ptr.p, out_dst.p, bt.dist.p, bt.sigma.p, bt.delta.p, W, level);
      SB_CHECK_LAUNCH();
    }
    SB_LAUNCH(k_bc_accum, div_up(N * 32, TPB), TPB, 0, s, N, st.visited.p, bt.dist.p, bt.delta.p, W, cent.p, reached.p);
    SB_CHECK_LAUNCH();
  }

  // centrality / (n * (n - 1.0)) with n as f64: n == 1 divides by zero like the reference
  const double n = (double)n_sources, norm = n * (n - 1.0);
  DevBuf<uint32_t> flag, pos; DevBuf<double> val;
  SB_TRY(flag.alloc(N + 1)); SB_TRY(pos.alloc(N + 1)); SB_TRY(val.alloc(N));
  SB_CUDA(cudaMemsetAsync(flag.p + N, 0, 4, s));
  SB_LAUNCH(k_bc_flags, div_up(N, TPB), TPB, 0, s, g->inv.p, cent.p, reached.p, N, norm, flag.p, val.p);
  SB_CHECK_LAUNCH();
  size_t need = 0;
  DevBuf<uint8_t> tmp;
  SB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, need, flag.p, pos.p, (int64_t)(N + 1), s));
  SB_TRY(tmp.alloc(need + 256));
  SB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, need, flag.p, pos.p, (int64_t)(N + 1), s));
  g_launches.fetch_add(2, std::memory_order_relaxed);
  uint32_t total = 0;
  SB_CUDA(cudaMemcpyAsync(&total, pos.p + N, 4, cudaMemcpyDeviceToHost, s));
  SB_CUDA(cudaStreamSynchronize(s));
  DevBuf<uint64_t> olo, ohi; DevBuf<double> oc;
  SB_TRY(olo.alloc(total)); SB_TRY(ohi.alloc(total)); SB_TRY(oc.alloc(total));
  SB_LAUNCH(k_ah_scatter, div_up(N, TPB), TPB, 0, s, flag.p, pos.p, val.p, g->id_lo.p, g->id_hi.p, N, (uint64_t)total, olo.p, ohi.p, oc.p);
  SB_CHECK_LAUNCH();
  SB_CUDA(cudaMemcpyAsync(id_lo, olo.p, (size_t)total * 8, cudaMemcpyDefault, s));
  SB_CUDA(cudaMemcpyAsync(id_hi, ohi.p, (size_t)total * 8, cudaMemcpyDefault, s));
  SB_CUDA(cudaMemcpyAsync(centrality, oc.p, (size_t)total * 8, cudaMemcpyDefault, s));
  SB_CUDA(cudaStreamSynchronize(s));
  *len = total;
  *max_dist = deepest;
  return SB200_OK;
}

}  // extern "C"
