// graph_bfs.cu -- bit-parallel multi-source BFS over the resident CSR (SURVEY 8(f) rank 4: the other graph kernels).
//
// Reference:
//   dijkstra_multi with unit edge costs            crates/core/src/webgraph/shortest_path.rs:57-105
//     raw_distances / raw_distances_with_max / raw_reversed_distances(_with_max)   :122-214
//   ApproxHarmonic::build                          crates/core/src/webgraph/centrality/approx_harmonic.rs:40-88
//     sample ceil(log2(n) / 0.3^2) nodes, one bounded shortest-path search per sample (max_dist 7), every reached
//     target gets += (1/dist) * n / (samples * (n - 1)) in f32
//
// All edge costs are 1, so the reference's Dijkstra is a breadth-first search.  Up to 64 searches run at once: bit b of a
// node's 64-bit word says "search b has reached this node".  One level = OR the frontier words of the in-neighbours
// (forward search, a pull over the destination-major CSR: no atomics on the row being built) or OR the row's frontier word
// into its in-neighbours (reversed search, atomicOr), then commit: new = next & ~visited.
// The cut-off reproduces dijkstra_multi's: the loop returns when it POPS a node with cost > max_dist, by which time every
// node at cost max_dist + 1 has already been inserted -- distances up to max_dist + 1 are reported.
#include "graph.cuh"

#ifndef SB200_EMU
#include <cub/cub.cuh>
#endif
#include <algorithm>
#include <vector>

namespace sb200 {

// seeds: rank (position in ascending id order) -> internal row through `inv`
__global__ void k_bfs_seed(const uint32_t* __restrict__ seed_rank, const uint32_t* __restrict__ seed_bit, uint32_t n, const uint32_t* __restrict__ inv,
                           unsigned long long* frontier, unsigned long long* visited) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t v = inv[seed_rank[i]];
  const unsigned long long b = 1ull << seed_bit[i];
  atomicOr(frontier + v, b); atomicOr(visited + v, b);
}
// forward level, long rows: one warp per <= CHUNK_EDGES work item, OR-reduce, one atomicOr per item
__global__ void __launch_bounds__(256) k_bfs_pull_items(uint64_t n_items, const uint32_t* __restrict__ item_row, const uint32_t* __restrict__ item_start,
    uint32_t warp_row_begin, const uint32_t* __restrict__ row_ptr, const uint32_t* __restrict__ col,
    const unsigned long long* __restrict__ frontier, unsigned long long* next) {
  const uint64_t item = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  if (item >= n_items) return;
  const uint32_t lane = threadIdx.x & 31, row = item_row[item];
  const uint32_t c = (uint32_t)item - item_start[row - warp_row_begin];
  const uint32_t e0 = row_ptr[row] + c * (uint32_t)CHUNK_EDGES, e1 = min(e0 + (uint32_t)CHUNK_EDGES, row_ptr[row + 1]);
  unsigned long long acc = 0;
  for (uint32_t e = e0 + lane; e < e1; e += 32) acc |= frontier[col[e]];
  for (int o = 16; o; o >>= 1) acc |= __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0 && acc) atomicOr(next + row, acc);
}
// forward level, short rows (<= QUAD_MAX_DEG in-edges): one thread per row
__global__ void k_bfs_pull_rows(uint64_t row_begin, uint64_t row_end, const uint32_t* __restrict__ row_ptr, const uint32_t* __restrict__ col,
                                const unsigned long long* __restrict__ frontier, unsigned long long* next) {
  const uint64_t row = row_begin + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (row >= row_end) return;
  unsigned long long acc = 0;
  for (uint32_t e = row_ptr[row]; e < row_ptr[row + 1]; e++) acc |= frontier[col[e]];
  if (acc) next[row] = acc;   // one writer per row in this kernel; long rows go through k_bfs_pull_items
}
// reversed level: the frontier word of row v flows to v's in-neighbours
__global__ void __launch_bounds__(256) k_bfs_push_items(uint64_t n_items, const uint32_t* __restrict__ item_row, const uint32_t* __restrict__ item_start,
    uint32_t warp_row_begin, const uint32_t* __restrict__ row_ptr, const uint32_t* __restrict__ col,
    const unsigned long long* __restrict__ frontier, unsigned long long* next) {
  const uint64_t item = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  if (item >= n_items) return;
  const uint32_t lane = threadIdx.x & 31, row = item_row[item];
  const unsigned long long f = frontier[row];
  if (!f) return;
  const uint32_t c = (uint32_t)item - item_start[row - warp_row_begin];
  const uint32_t e0 = row_ptr[row] + c * (uint32_t)CHUNK_EDGES, e1 = min(e0 + (uint32_t)CHUNK_EDGES, row_ptr[row + 1]);
  for (uint32_t e = e0 + lane; e < e1; e += 32) atomicOr(next + col[e], f);
}
__global__ void k_bfs_push_rows(uint64_t row_begin, uint64_t row_end, const uint32_t* __restrict__ row_ptr, const uint32_t* __restrict__ col,
                                const unsigned long long* __restrict__ frontier, unsigned long long* next) {
  const uint64_t row = row_begin + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (row >= row_end) return;
  const unsigned long long f = frontier[row];
  if (!f) return;
  for (uint32_t e = row_ptr[row]; e < row_ptr[row + 1]; e++) atomicOr(next + col[e], f);
}
// commit a level: the searches that reach v for the first time.  dist_out (nullable): [n_bits][N] in rank order;
// cent (nullable): += popcount(new) * term (ApproxHarmonic's accumulation, kept in f64)
__global__ void k_bfs_commit(uint64_t N, const uint32_t* __restrict__ perm, unsigned long long* next, unsigned long long* visited,
                             unsigned long long* frontier, uint32_t level, uint8_t* dist_out, uint32_t n_bits, double* cent, double term,
                             unsigned long long* any) {
  const uint64_t v = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  unsigned long long nb = 0;
  if (v < N) {
    nb = next[v] & ~visited[v];
    next[v] = 0;
    frontier[v] = nb;
    if (nb) {
      visited[v] |= nb;
      if (cent) cent[v] += (double)__popcll(nb) * term;
      if (dist_out) {
        const uint64_t r = perm[v];
        unsigned long long m = nb;
        while (m) { const int b = __ffsll((long long)m) - 1; m &= m - 1; if ((uint32_t)b < n_bits) dist_out[(uint64_t)b * N + r] = (uint8_t)level; }
      }
    }
  }
  if (__any_sync(0xffffffffu, nb != 0) && (threadIdx.x & 31) == 0) atomicOr(any, 1ull);
}
__global__ void k_bfs_dist_init(uint64_t n, uint8_t* d) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) d[i] = 255;
}
__global__ void k_bfs_dist_seed(const uint32_t* __restrict__ seed_rank, const uint32_t* __restrict__ seed_bit, uint32_t n, uint64_t N, uint8_t* d) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) d[(uint64_t)seed_bit[i] * N + seed_rank[i]] = 0;
}
// u128 id -> rank by binary search over the ascending (hi, lo) arrays; 0xFFFFFFFF when the id is not a node
__global__ void k_id_to_rank(const uint64_t* __restrict__ q_lo, const uint64_t* __restrict__ q_hi, uint32_t n, const uint64_t* __restrict__ id_lo,
                             const uint64_t* __restrict__ id_hi, uint64_t N, uint32_t* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t lo = q_lo[i], hi = q_hi[i];
  uint64_t a = 0, b = N;
  while (a < b) {
    const uint64_t m = (a + b) >> 1;
    const bool less = id_hi[m] < hi || (id_hi[m] == hi && id_lo[m] < lo);
    if (less) a = m + 1; else b = m;
  }
  out[i] = (a < N && id_hi[a] == hi && id_lo[a] == lo) ? (uint32_t)a : 0xFFFFFFFFu;
}
__global__ void k_ah_flags(const uint32_t* __restrict__ inv, const double* __restrict__ cent, uint64_t N, uint32_t* flag, double* val) {
  const uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (r >= N) return;
  const double c = cent[inv[r]];
  flag[r] = c != 0.0 ? 1u : 0u;   // the reference's map only holds targets that were reached
  val[r] = c;
}
__global__ void k_ah_scatter(const uint32_t* __restrict__ flag, const uint32_t* __restrict__ pos, const double* __restrict__ val,
                             const uint64_t* __restrict__ id_lo, const uint64_t* __restrict__ id_hi, uint64_t N, uint64_t cap, uint64_t* out_lo,
                             uint64_t* out_hi, double* out_c) {
  const uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (r >= N || !flag[r]) return;
  const uint32_t p = pos[r];
  if (p >= cap) return;
  out_lo[p] = id_lo[r]; out_hi[p] = id_hi[r]; out_c[p] = val[r];
}

// one batch of <= 64 searches; levels 1 .. max_level are committed (max_level == 0: until no search makes progress)
static int bfs_batch(sb200_graph* g, BfsState& st, uint32_t n_seeds, uint32_t n_bits, uint32_t max_level, bool reversed, uint8_t* dist_dev,
                     double* cent, const std::vector<double>& term_of_level) {
  cudaStream_t s = g->stream;
  const uint64_t N = g->N;
  SB_CUDA(cudaMemsetAsync(st.frontier.p, 0, N * 8, s)); SB_CUDA(cudaMemsetAsync(st.next.p, 0, N * 8, s)); SB_CUDA(cudaMemsetAsync(st.visited.p, 0, N * 8, s));
  SB_LAUNCH(k_bfs_seed, div_up(n_seeds, 256), 256, 0, s, st.seed_rank.p, st.seed_bit.p, n_seeds, g->inv.p, st.frontier.p, st.visited.p);
  SB_CHECK_LAUNCH();
  const uint64_t nq = g->quad_row_end - g->quad_row_begin;
  for (uint32_t level = 1; max_level == 0 || level <= max_level; level++) {
    if (level > 254) break;   // distances are u8 in the reference
    if (g->n_items) {
      if (reversed) SB_LAUNCH(k_bfs_push_items, div_up(g->n_items * 32, 256), 256, 0, s, g->n_items, g->item_row.p, g->item_start.p, (uint32_t)g->warp_row_begin,
                              g->row_ptr.p, g->col.p, st.frontier.p, st.next.p);
      else SB_LAUNCH(k_bfs_pull_items, div_up(g->n_items * 32, 256), 256, 0, s, g->n_items, g->item_row.p, g->item_start.p, (uint32_t)g->warp_row_begin,
                     g->row_ptr.p, g->col.p, st.frontier.p, st.next.p);
      SB_CHECK_LAUNCH();
    }
    if (nq) {
      if (reversed) SB_LAUNCH(k_bfs_push_rows, div_up(nq, 256), 256, 0, s, g->quad_row_begin, g->quad_row_end, g->row_ptr.p, g->col.p, st.frontier.p, st.next.p);
      else SB_LAUNCH(k_bfs_pull_rows, div_up(nq, 256), 256, 0, s, g->quad_row_begin, g->quad_row_end, g->row_ptr.p, g->col.p, st.frontier.p, st.next.p);
      SB_CHECK_LAUNCH();
    }
    SB_CUDA(cudaMemsetAsync(st.any.p, 0, 8, s));
    const double term = level < term_of_level.size() ? term_of_level[level] : 0.0;
    SB_LAUNCH(k_bfs_commit, div_up(N, 256), 256, 0, s, N, g->perm.p, st.next.p, st.visited.p, st.frontier.p, level, dist_dev, n_bits, cent, term, st.any.p);
    SB_CHECK_LAUNCH();
    unsigned long long any = 0;
    SB_CUDA(cudaMemcpyAsync(&any, st.any.p, 8, cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaStreamSynchronize(s));
    if (!any) break;
  }
  return SB200_OK;
}

int bfs_prepare(sb200_graph* g, BfsState& st, const uint64_t* src_lo, const uint64_t* src_hi, uint32_t n_sources, std::vector<uint32_t>& ranks) {
  cudaStream_t s = g->stream;
  if (g->world != 1) SB_FAIL(SB200_ESTATE, "graph searches run on single-rank handles");
  const uint64_t N = g->N;
  SB_TRY(st.frontier.alloc(std::max<uint64_t>(N, 1))); SB_TRY(st.next.alloc(std::max<uint64_t>(N, 1))); SB_TRY(st.visited.alloc(std::max<uint64_t>(N, 1)));
  SB_TRY(st.any.alloc(1));
  ranks.assign(n_sources, 0xFFFFFFFFu);
  if (!n_sources || !N) return SB200_OK;
  DevBuf<uint64_t> qlo, qhi; DevBuf<uint32_t> out;
  SB_TRY(qlo.alloc(n_sources)); SB_TRY(qhi.alloc(n_sources)); SB_TRY(out.alloc(n_sources));
  SB_CUDA(cudaMemcpyAsync(qlo.p, src_lo, (size_t)n_sources * 8, cudaMemcpyDefault, s));
  SB_CUDA(cudaMemcpyAsync(qhi.p, src_hi, (size_t)n_sources * 8, cudaMemcpyDefault, s));
  SB_LAUNCH(k_id_to_rank, div_up(n_sources, 256), 256, 0, s, qlo.p, qhi.p, n_sources, g->id_lo.p, g->id_hi.p, N, out.p);
  SB_CHECK_LAUNCH();
  SB_CUDA(cudaMemcpyAsync(ranks.data(), out.p, (size_t)n_sources * 4, cudaMemcpyDeviceToHost, s));
  SB_CUDA(cudaStreamSynchronize(s));
  return SB200_OK;
}

}  // namespace sb200
using namespace sb200;

extern "C" {

int sb200_graph_distances(sb200_graph* g, const uint64_t* src_lo, const uint64_t* src_hi, const uint32_t* src_group, uint32_t n_sources,
                          uint32_t n_groups, uint32_t max_dist, int reversed, uint8_t* dist_out) {
  if (!g) SB_FAIL(SB200_EINVAL, "NULL graph handle");
  SB_CUDA(cudaSetDevice(g->device));
  if (!dist_out || (n_sources && (!src_lo || !src_hi))) SB_FAIL(SB200_EINVAL, "NULL argument");
  if (n_groups == 0 || n_groups > 64) SB_FAIL(SB200_ERANGE, "n_groups %u outside [1,64]", n_groups);
  if (max_dist > 253) SB_FAIL(SB200_ERANGE, "max_dist %u > 253 (distances are u8; 0 = unbounded)", max_dist);
  cudaStream_t s = g->stream;
  const uint64_t N = g->N;
  if (!N) return SB200_OK;
  PoolScope scope(s);
  BfsState st;
  std::vector<uint32_t> ranks;
  SB_TRY(bfs_prepare(g, st, src_lo, src_hi, n_sources, ranks));
  std::vector<uint32_t> sr, sbit;
  for (uint32_t i = 0; i < n_sources; i++) {
    const uint32_t grp = src_group ? src_group[i] : i;
    if (grp >= n_groups) SB_FAIL(SB200_EINVAL, "source %u: group %u >= %u", i, grp, n_groups);
    if (ranks[i] == 0xFFFFFFFFu) continue;   // a source that is not a node of the graph reaches nothing (but itself, which is not a node)
    sr.push_back(ranks[i]); sbit.push_back(grp);
  }
  DevBuf<uint8_t> dist;
  SB_TRY(dist.alloc((size_t)n_groups * N));
  SB_LAUNCH(k_bfs_dist_init, div_up((uint64_t)n_groups * N, 256), 256, 0, s, (uint64_t)n_groups * N, dist.p);
  SB_CHECK_LAUNCH();
  const uint32_t n_seeds = (uint32_t)sr.size();
  if (n_seeds) {
    SB_TRY(st.seed_rank.alloc(n_seeds)); SB_TRY(st.seed_bit.alloc(n_seeds));
    SB_CUDA(cudaMemcpyAsync(st.seed_rank.p, sr.data(), (size_t)n_seeds * 4, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(st.seed_bit.p, sbit.data(), (size_t)n_seeds * 4, cudaMemcpyHostToDevice, s));
    SB_LAUNCH(k_bfs_dist_seed, div_up(n_seeds, 256), 256, 0, s, st.seed_rank.p, st.seed_bit.p, n_seeds, N, dist.p);
    SB_CHECK_LAUNCH();
    // dijkstra_multi returns when it pops cost > max_dist: distances up to max_dist + 1 have been inserted by then
    SB_TRY(bfs_batch(g, st, n_seeds, n_groups, max_dist ? max_dist + 1 : 0, reversed != 0, dist.p, nullptr, std::vector<double>()));
  }
  SB_CUDA(cudaMemcpyAsync(dist_out, dist.p, (size_t)n_groups * N, cudaMemcpyDefault, s));
  SB_CUDA(cudaStreamSynchronize(s));
  return SB200_OK;
}

int sb200_approx_harmonic(sb200_graph* g, const uint64_t* src_lo, const uint64_t* src_hi, uint32_t n_sources, uint32_t max_dist,
                          uint64_t num_nodes, uint64_t* id_lo, uint64_t* id_hi, double* centrality, uint64_t cap, uint64_t* len) {
  if (!g) SB_FAIL(SB200_EINVAL, "NULL graph handle");
  SB_CUDA(cudaSetDevice(g->device));
  if (!len || (n_sources && (!src_lo || !src_hi))) SB_FAIL(SB200_EINVAL, "NULL argument");
  if (centrality && (!id_lo || !id_hi)) SB_FAIL(SB200_EINVAL, "id outputs are NULL");
  if (max_dist == 0 || max_dist > 253) SB_FAIL(SB200_ERANGE, "max_dist %u outside [1,253]", max_dist);
  cudaStream_t s = g->stream;
  const uint64_t N = g->N;
  *len = 0;
  if (!N || !n_sources) return SB200_OK;
  if (num_nodes == 0) num_nodes = N;
  PoolScope scope(s);
  BfsState st;
  std::vector<uint32_t> ranks;
  SB_TRY(bfs_prepare(g, st, src_lo, src_hi, n_sources, ranks));
  // norm = num_nodes as f32 / (num_samples as f32 * (num_nodes as f32 - 1.0)); term(dist) = (1.0 / dist as f32) * norm  -- all f32
  const float nn = (float)num_nodes;
  const float norm = nn / ((float)n_sources * (nn - 1.0f));
  std::vector<double> term(max_dist + 2, 0.0);
  for (uint32_t d = 1; d <= max_dist + 1; d++) term[d] = (double)((1.0f / (float)d) * norm);
  DevBuf<double> cent;
  SB_TRY(cent.alloc(N));
  SB_CUDA(cudaMemsetAsync(cent.p, 0, N * 8, s));
  SB_TRY(st.seed_rank.alloc(64)); SB_TRY(st.seed_bit.alloc(64));
  for (uint32_t base = 0; base < n_sources; base += 64) {
    std::vector<uint32_t> sr, sbit;
    for (uint32_t i = base; i < std::min(n_sources, base + 64); i++) if (ranks[i] != 0xFFFFFFFFu) { sr.push_back(ranks[i]); sbit.push_back(i - base); }
    if (sr.empty()) continue;
    SB_CUDA(cudaMemcpyAsync(st.seed_rank.p, sr.data(), sr.size() * 4, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(st.seed_bit.p, sbit.data(), sbit.size() * 4, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaStreamSynchronize(s));   // sr / sbit go out of scope
    SB_TRY(bfs_batch(g, st, (uint32_t)sr.size(), 64, max_dist + 1, false, nullptr, cent.p, term));
  }
  DevBuf<uint32_t> flag, pos; DevBuf<double> val;
  SB_TRY(flag.alloc(N + 1)); SB_TRY(pos.alloc(N + 1)); SB_TRY(val.alloc(N));
  SB_CUDA(cudaMemsetAsync(flag.p + N, 0, 4, s));
  SB_LAUNCH(k_ah_flags, div_up(N, 256), 256, 0, s, g->inv.p, cent.p, N, flag.p, val.p);
  SB_CHECK_LAUNCH();
  size_t need = 0;
  SB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, need, flag.p, pos.p, (int64_t)(N + 1), s));
  if (g->cub_tmp.n < need) SB_TRY(g->cub_tmp.alloc(need + 256));
  SB_CUDA(cub::DeviceScan::ExclusiveSum(g->cub_tmp.p, need, flag.p, pos.p, (int64_t)(N + 1), s));
  g_launches.fetch_add(2, std::memory_order_relaxed);
  uint32_t total = 0;
  SB_CUDA(cudaMemcpyAsync(&total, pos.p + N, 4, cudaMemcpyDeviceToHost, s));
  SB_CUDA(cudaStreamSynchronize(s));
  *len = total;
  const uint64_t k = std::min<uint64_t>(total, cap);
  if (!centrality || k == 0) return SB200_OK;
  DevBuf<uint64_t> olo, ohi; DevBuf<double> oc;
  SB_TRY(olo.alloc(k)); SB_TRY(ohi.alloc(k)); SB_TRY(oc.alloc(k));
  SB_LAUNCH(k_ah_scatter, div_up(N, 256), 256, 0, s, flag.p, pos.p, val.p, g->id_lo.p, g->id_hi.p, N, k, olo.p, ohi.p, oc.p);
  SB_CHECK_LAUNCH();
  SB_CUDA(cudaMemcpyAsync(id_lo, olo.p, k * 8, cudaMemcpyDefault, s));
  SB_CUDA(cudaMemcpyAsync(id_hi, ohi.p, k * 8, cudaMemcpyDefault, s));
  SB_CUDA(cudaMemcpyAsync(centrality, oc.p, k * 8, cudaMemcpyDefault, s));
  SB_CUDA(cudaStreamSynchronize(s));
  return SB200_OK;
}

}  // extern "C"
