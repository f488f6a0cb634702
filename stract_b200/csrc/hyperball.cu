// hyperball.cu -- the HyperBall iteration on the device (hot path 1).
//
// Reference semantics (crates/core/src/webgraph/centrality/harmonic.rs):
//   update_all_counters  :116-157   for every kept edge u->v with u in the changed set:
//                                   if any(old[u][i] > new[v][i]) { new[v].merge(old[u]); mark v }
//   update_changed_counters :75-114 same, driven from the exact changed set through forward links
//   update_centralities  :159-176   score[v] += (size(new[v]) -sat size(old[v])) as f64 / (t+1)  (Kahan)
//   Counters::step       :210-212   old = new.clone()
// All branches compute the synchronous update new[v] = max(old[v], max_{u->v, u changed} old[u]);
// merging an unchanged u is a no-op (it was merged the iteration after it last changed), which is
// why the reference may use a Bloom filter for the changed set and why the dense kernel below may
// skip the frontier test altogether.
//
// Device formulation
//   * registers live in two N x 64 B arrays (ping-pong).  Row v of the "new" array is rewritten only
//     if v changed now or changed in the previous iteration (it is then two iterations stale);
//     every other row is already equal in both arrays, so `old = new.clone()` costs nothing.
//   * pull kernels (destination-major CSR, one writer per row, no atomics on registers):
//       k_pull_quad : rows with in-degree <= 32, 4 lanes per row (16 B of the 64-B counter each)
//       k_pull_warp : longer rows cut into 1024-edge work items, one warp per item: the 32 source
//                     indices of a batch are loaded coalesced, each quad of lanes gathers one 64-B
//                     counter (4 x LDG.128), byte-wise max with __vmaxu4, xor-shuffle reduce over
//                     the 8 quads; rows spanning several items go through a partial buffer + k_pull_merge
//     DENSE variant gathers every in-neighbour; FRONTIER variant tests the changed bitmap first; SEED variant (iteration
//     0) gathers every in-neighbour's 2-B seed instead of its 64-B row: a reset counter has one non-zero register.
//     Every gather of a source below the L1 hub budget (the highest in-degrees: rows are numbered by in-degree) goes
//     through L1 with evict_last, every other one around L1 (ld_gather_u4).  The default budget is every row: at C2 no
//     smaller budget was faster (DESIGN section 6).
//   * push kernel (source-major CSR) for small frontiers: the frontier's out-edges in equal contiguous tiles per warp,
//     half-warp per out-edge, 32-bit CAS max.
//   * k_finalize: per changed node, HyperLogLog<64>::size() in the reference's exact f64 operation
//     order (sequential sum over registers 0..63, no FMA), saturating difference against the cached
//     size(old), KahanSum update; nodes that changed in the previous iteration but not now get the
//     reference's "+= 0.0" (it is idempotent after one application, so skipping the other N-1 zero
//     adds is bit-exact).
// Roofline: HBM.  Algorithmic bytes per iteration: 68 B x E_active + 132 B x N_written + 40 B x N_changed
// (iteration 0: 6 B per edge instead of 68, the index and a 2-B seed).
#include <chrono>
#include "graph.cuh"
#include "../../include/sb200_hll_tables.h"

#ifndef SB200_EMU
#include <cub/cub.cuh>
#endif
#include <algorithm>
#include <cmath>
#include <cstdlib>

namespace sb200 {

struct HllTables {
  double raw[SB200_HLL_P5_LEN];
  double bias[SB200_HLL_P5_LEN];
  double lc[65];  // lc[v] = 64*ln(64/v), host libm (matches the reference's f64::ln), lc[0] unused
};
__constant__ HllTables c_tab;
static bool g_tab_loaded[64] = {false};

static int pulls_prefer_l1();
// once per device: the HyperLogLog tables, and the pull kernels' cache configuration
int load_tables(int device) {
  if (device >= 0 && device < 64 && g_tab_loaded[device]) return SB200_OK;
  static HllTables h;
  for (int i = 0; i < SB200_HLL_P5_LEN; i++) { h.raw[i] = SB200_HLL_RAW_P5[i]; h.bias[i] = SB200_HLL_BIAS_P5[i]; }
  h.lc[0] = 0.0;
  for (int v = 1; v <= 64; v++) h.lc[v] = 64.0 * std::log(64.0 / (double)v);  // hyperloglog.rs:4472-4476
  SB_CUDA(cudaMemcpyToSymbol(c_tab, &h, sizeof(h)));
  SB_TRY(pulls_prefer_l1());
  if (device >= 0 && device < 64) g_tab_loaded[device] = true;
  return SB200_OK;
}

// ---- HyperLogLog<64>::size(), crates/core/src/hyperloglog.rs:4484-4516, bit-exact -----------------
// `tab` points to a shared-memory copy of c_tab (divergent indexing into __constant__ serialises).
__device__ __forceinline__ double pow2_neg(uint32_t k) {  // ONE_OVER_POWER_OF_TWO[k] == 2^-k
  return __longlong_as_double((long long)(1023 - (int)k) << 52);
}
__device__ uint64_t hll64_size(const uint32_t w[16], const HllTables* tab) {
  double sum = 0.0;
  int zeros = 0;
#pragma unroll
  for (int i = 0; i < 16; i++) {
#pragma unroll
    for (int b = 0; b < 4; b++) {
      uint32_t r = (w[i] >> (8 * b)) & 0xFFu;
      sum = __dadd_rn(sum, pow2_neg(r));
      zeros += (r == 0);
    }
  }
  const double z = __ddiv_rn(1.0, sum);
  const double e = __dmul_rn(0.709 * 4096.0, z);  // am() * m.powi(2) * z, left-assoc; 0.709*2^12 is exact
  double e_star = e;
  if (e <= 320.0) {
    // estimate_bias(e, 6): tables [b-1-4] = "precision 5"; Rust >= 1.82 binary_search_by
    const int LEN = SB200_HLL_P5_LEN;
    int size = LEN, base = 0;
    while (size > 1) {
      int half = size >> 1, mid = base + half;
      base = (tab->raw[mid] > e) ? base : mid;
      size -= half;
    }
    int r = base;
    if (!(tab->raw[base] == e)) r = base + (tab->raw[base] < e ? 1 : 0);
    if (r == LEN) r = LEN - 1;
    int il = r, ir = (r < LEN - 1) ? r + 1 : -1;
    double bsum = 0.0;
#pragma unroll 1
    for (int k = 0; k < 6; k++) {
      bool right;
      int idx;
      if (il >= 0 && ir >= 0) {
        double dl = fabs(__dsub_rn(tab->raw[il], e)), dr = fabs(__dsub_rn(tab->raw[ir], e));
        right = dr < dl;
        idx = right ? ir : il;
      } else if (il >= 0) { right = false; idx = il; }
      else { right = true; idx = ir; }
      bsum = __dadd_rn(bsum, tab->bias[idx]);
      if (right) ir = (idx < LEN - 1) ? idx + 1 : -1;
      else il = (idx > 0) ? idx - 1 : -1;
    }
    e_star = __dsub_rn(e, __ddiv_rn(bsum, 6.0));
  }
  const double h = (zeros != 0) ? tab->lc[zeros] : e_star;
  const double pick = (h <= 40.0) ? h : e_star;  // threshold(b=6) = 40
  // Rust `as usize`: saturating, NaN -> 0
  if (!(pick == pick) || pick <= 0.0) return 0ull;
  if (pick >= 18446744073709551616.0) return 0xFFFFFFFFFFFFFFFFull;
  return (uint64_t)__double2ull_rz(pick);
}

__device__ __forceinline__ void kahan_add(double& sum, double& err, double rhs) {  // kahan_sum.rs:46-53
  const double y = __dsub_rn(rhs, err);
  const double t = __dadd_rn(sum, y);
  err = __dsub_rn(__dsub_rn(t, sum), y);
  sum = t;
}

// ---- init: counters seeded with the node's own id (low 64 bits), harmonic.rs:53-73 ------------------
// A freshly seeded counter has one non-zero register: j = hash >> 58 holds p = clz(hash << 6) + 1 (1..65).  The seed
// j | p << 8 is all of it, and iteration 0 reads 2 B per source instead of 64 (see the SEED pull variants).
// seed_slice expands a seed into the 16-B slice `sub` of its row (registers 16 sub .. 16 sub + 15).
__device__ __forceinline__ uint4 seed_slice(uint32_t s, uint32_t sub) {
  const uint32_t j = s & 63u;
  const uint32_t v = ((j >> 4) == sub) ? (s >> 8) << (8 * (j & 3u)) : 0u;
  const uint32_t w = (j >> 2) & 3u;
  return make_uint4(w == 0u ? v : 0u, w == 1u ? v : 0u, w == 2u ? v : 0u, w == 3u ? v : 0u);
}
// One quad of lanes per node: lane q stores the 16-B slice q of both register rows, so that a warp writes 8 whole rows (512 B)
// per store instruction.  size() of a freshly seeded counter needs no register sum: with one non-zero register, zeros = 63
// and linear counting decides (h = lc[63] = 64 ln(64/63) = 1.008 is below the threshold 40, the `pick` of hll64_size), so
// it is (usize) lc[63] = 1 for every node.
__global__ void k_hb_init(const uint64_t* __restrict__ id_lo, const uint32_t* __restrict__ perm, uint64_t N,
                          uint4* r0, uint4* r1, uint16_t* seed, uint64_t* size_cache, double* ksum, double* kerr) {
  const uint64_t gt = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const uint64_t v = gt >> 2;
  const uint32_t q = (uint32_t)gt & 3u;
  if (v >= N) return;
  const uint64_t hash = id_lo[perm[v]] * 11400714819323198549ull;  // FastHasher hyperloglog.rs:4311-4313
  const uint32_t j = (uint32_t)(hash >> 58);
  const uint64_t wv = hash << 6;
  const uint32_t p = (wv == 0 ? 64u : (uint32_t)__clzll((long long)wv)) + 1u;
  const uint32_t s = j | p << 8;
  const uint4 x = seed_slice(s, q);
  r0[v * 4 + q] = x; r1[v * 4 + q] = x;
  if (q == 0) { seed[v] = (uint16_t)s; size_cache[v] = (uint64_t)__double2ull_rz(c_tab.lc[63]); }
  else if (q == 1) ksum[v] = 0.0;
  else if (q == 2) kerr[v] = 0.0;
}
__global__ void k_bm_fill(uint32_t* bm, uint64_t N, uint64_t words) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= words) return;
  uint64_t first = i * 32;
  uint32_t m = 0xFFFFFFFFu;
  if (first + 32 > N) m = (N > first) ? ((1u << (N - first)) - 1u) : 0u;
  bm[i] = m;
}

// Fused exchange: a produced row is stored into the local `new` array AND, over NVLink peer memory, into every
// other rank's replica of it (one writer per row, so plain 16-B stores; the changed bit goes through a
// system-scope atomic OR).  This replaces the per-iteration all-gather: the transfer of a row overlaps the
// gathers of the rows still being computed, and rows that did not change never cross the link.
// sharded handles: destination rows are owned in interleaved blocks of 32 (block b -> rank b % world)
__device__ __forceinline__ bool owned_row(const PeerOut& o, uint32_t row) {
  return o.world <= 1u || ((row >> 5) % o.world) == o.rank;
}
// Subscriber filter: a peer that has no in-edge from `row` never gathers it, so the row is stored only into the
// replicas of the ranks named in its subscriber mask (at C2 size 69 % / 55 % / 42 % of the (row, peer) pairs at
// 2 / 4 / 8 ranks).  A non-subscriber's copy of the row simply stays at its initial value and is never read.
__device__ __forceinline__ void publish_row(uint4* __restrict__ newr, uint32_t* __restrict__ bm_cur, const PeerOut& peers,
                                            uint32_t row, uint32_t sub, uint4 acc, bool write, bool changed) {
  if (write) newr[(uint64_t)row * 4 + sub] = acc;
  if (changed && sub == 0) atomicOr(bm_cur + (row >> 5), 1u << (row & 31));
  if (!write || peers.n == 0) return;
  const uint32_t want = peers.sub ? __ldg(peers.sub + row) : 0xFFFFFFFFu;
  for (int p = 0; p < peers.n; p++) {
    if ((want >> peers.prank[p]) & 1u) peers.newr[p][(uint64_t)row * 4 + sub] = acc;
    // the changed bit is NOT pushed per row: a 32-row block has one owner, so k_publish_bitmap copies the owner's
    // finished bitmap words to the peers with plain stores (per-row remote atomics would be one per changed row,
    // peer and iteration)
  }
}

__device__ __forceinline__ bool bm_test(const uint32_t* __restrict__ bm, uint32_t v) {
  return (__ldg(bm + (v >> 5)) >> (v & 31)) & 1u;
}

// ---- pull, short rows: 4 lanes per destination row ----------------------------------------------------
// SEED (iteration 0 only, see hb_step_launch): every row of `oldr` is the one-hot row of its seed, so the own row and
// the sources are built from seed[] (2 B per source, L2-resident) and `oldr` is not read.
// l1_hub: sources below it are hubs, gathered through L1 (ld_gather_u4); the SEED variant's cached 2-B loads ignore it.
template <bool FRONTIER, bool SEED>
__device__ __forceinline__ void quad_rows(uint64_t row, bool live, uint32_t sub, uint32_t lane,
    const uint32_t* __restrict__ row_ptr, const uint32_t* __restrict__ col,
    const uint4* __restrict__ oldr, const uint16_t* __restrict__ seed, uint4* __restrict__ newr,
    const uint32_t* __restrict__ bm_prev, uint32_t* __restrict__ bm_cur, const PeerOut& peers, uint32_t l1_hub) {
  static_assert(!(FRONTIER && SEED), "the seed iteration gathers every source");
  const uint32_t e0 = live ? row_ptr[row] : 0u, e1 = live ? row_ptr[row + 1] : 0u;
  const uint4 own = SEED ? seed_slice(__ldg(seed + row), sub)
                         : ld_gather_u4(oldr + row * 4 + sub, row < l1_hub);
  uint4 acc = own;
  // lane `sub` fetches source index e+sub (one 16-B request per quad per 4 edges, prefetched one step ahead)
  // and the quad shares the four indices by shuffle; an out-of-range or (FRONTIER) unchanged source is
  // redirected to the row itself, which is a no-op under max.
  const unsigned qmask = 0xFu << (lane & ~3u);
  const uint32_t self = (uint32_t)row;
  uint32_t nxt = (e0 + sub < e1) ? ld_stream_u32(col + e0 + sub) : self;
  if (SEED) {
    // the seed of step k is loaded during step k-1 and the index of step k+1 with it, so that one seed and one index
    // load per lane are in flight while the quad folds in the previous four seeds
    uint32_t sn = __ldg(seed + nxt);
    nxt = (e0 + 4 + sub < e1) ? ld_stream_u32(col + e0 + 4 + sub) : self;
    for (uint32_t e = e0; e < e1; e += 4) {
      const uint32_t mine = sn;
      sn = __ldg(seed + nxt);
      nxt = (e + 8 + sub < e1) ? ld_stream_u32(col + e + 8 + sub) : self;
      const uint32_t s0 = __shfl_sync(qmask, mine, 0, 4);
      const uint32_t s1 = __shfl_sync(qmask, mine, 1, 4);
      const uint32_t s2 = __shfl_sync(qmask, mine, 2, 4);
      const uint32_t s3 = __shfl_sync(qmask, mine, 3, 4);
      acc = vmax_u8x16(vmax_u8x16(acc, seed_slice(s0, sub)),
                       vmax_u8x16(vmax_u8x16(seed_slice(s1, sub), seed_slice(s2, sub)), seed_slice(s3, sub)));
    }
  } else
  for (uint32_t e = e0; e < e1; e += 4) {
    uint32_t mine = nxt;
    nxt = (e + 4 + sub < e1) ? ld_stream_u32(col + e + 4 + sub) : self;
    if (FRONTIER) mine = bm_test(bm_prev, mine) ? mine : self;
    const uint32_t i0 = __shfl_sync(qmask, mine, 0, 4);
    const uint32_t i1 = __shfl_sync(qmask, mine, 1, 4);
    const uint32_t i2 = __shfl_sync(qmask, mine, 2, 4);
    const uint32_t i3 = __shfl_sync(qmask, mine, 3, 4);
    const uint4 v0 = ld_gather_u4(oldr + (uint64_t)i0 * 4 + sub, i0 < l1_hub);
    const uint4 v1 = ld_gather_u4(oldr + (uint64_t)i1 * 4 + sub, i1 < l1_hub);
    const uint4 v2 = ld_gather_u4(oldr + (uint64_t)i2 * 4 + sub, i2 < l1_hub);
    const uint4 v3 = ld_gather_u4(oldr + (uint64_t)i3 * 4 + sub, i3 < l1_hub);
    acc = vmax_u8x16(vmax_u8x16(acc, v0), vmax_u8x16(vmax_u8x16(v1, v2), v3));
  }
  const unsigned ball = __ballot_sync(0xffffffffu, ne_u4(acc, own));
  const bool changed = ((ball >> (lane & ~3u)) & 0xFu) != 0u;
  if (!live) return;
  publish_row(newr, bm_cur, peers, (uint32_t)row, sub, acc, changed || bm_test(bm_prev, (uint32_t)row), changed);
}

template <bool FRONTIER, bool SEED>
__global__ void __launch_bounds__(256, 7) k_pull_quad(uint64_t row_begin, uint64_t row_end,
    const uint32_t* __restrict__ row_ptr, const uint32_t* __restrict__ col,
    const uint4* __restrict__ oldr, const uint16_t* __restrict__ seed, uint4* __restrict__ newr,
    const uint32_t* __restrict__ bm_prev, uint32_t* __restrict__ bm_cur, const PeerOut peers, uint32_t l1_hub) {
  const uint64_t gt = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const uint32_t sub = threadIdx.x & 3;
  const uint32_t lane = threadIdx.x & 31;
  uint64_t row = row_begin + (gt >> 2);
  bool live = row < row_end;
  if (!live) row = row_end - 1;  // keep the warp converged; results of dead quads are discarded
  live = live && owned_row(peers, (uint32_t)row);
  if (__ballot_sync(0xffffffffu, live) == 0u) return;  // none of this warp's rows belongs to this rank
  quad_rows<FRONTIER, SEED>(row, live, sub, lane, row_ptr, col, oldr, seed, newr, bm_prev, bm_cur, peers, l1_hub);
}

// Sharded handles with the fused exchange: the short rows are most of the rows, so this kernel carries most of the
// stores into the peers' replicas -- it is bound by NVLink, not by HBM, while k_pull_warp is the opposite.  This variant
// is a small persistent grid (a few CTAs per SM) that walks the OWNED 32-row blocks only (4 warps per block), so that it can
// sit next to k_pull_warp on a second, higher-priority stream: link traffic of the short rows under the gathers of the long ones.
template <bool FRONTIER, bool SEED>
__global__ void __launch_bounds__(256, 4) k_pull_quad_owned(uint64_t row_begin, uint64_t row_end, uint64_t first_block, uint64_t n_tasks,
    const uint32_t* __restrict__ row_ptr, const uint32_t* __restrict__ col,
    const uint4* __restrict__ oldr, const uint16_t* __restrict__ seed, uint4* __restrict__ newr,
    const uint32_t* __restrict__ bm_prev, uint32_t* __restrict__ bm_cur, const PeerOut peers, uint32_t l1_hub) {
  const uint32_t sub = threadIdx.x & 3, lane = threadIdx.x & 31;
  const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
  for (uint64_t task = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; task < n_tasks; task += warps) {
    const uint64_t block = first_block + (task >> 2) * peers.world;
    uint64_t row = block * 32 + (task & 3) * 8 + (lane >> 2);
    const bool live = row >= row_begin && row < row_end;
    if (!live) row = row_begin;
    if (__ballot_sync(0xffffffffu, live) == 0u) continue;
    quad_rows<FRONTIER, SEED>(row, live, sub, lane, row_ptr, col, oldr, seed, newr, bm_prev, bm_cur, peers, l1_hub);
  }
}

// ---- pull, long rows: one warp per <=CHUNK_EDGES work item ---------------------------------------------
template <bool FRONTIER, bool LISTED, bool SEED>
// 8 CTAs/SM (<= 32 registers): at full scale the gathers are DRAM-latency bound and the kernel's speed tracks the
// number of resident warps
__global__ void __launch_bounds__(256, 8) k_pull_warp(uint64_t n_items, uint64_t first_multi_free_item,
    const uint32_t* __restrict__ item_list, const uint32_t* __restrict__ item_row, const uint32_t* __restrict__ item_start, uint32_t warp_row_begin,
    const uint32_t* __restrict__ row_ptr, const uint32_t* __restrict__ col,
    const uint4* __restrict__ oldr, const uint16_t* __restrict__ seed, uint4* __restrict__ newr, uint4* __restrict__ partial,
    const uint32_t* __restrict__ bm_prev, uint32_t* __restrict__ bm_cur, const PeerOut peers, uint32_t l1_hub) {
  static_assert(!(FRONTIER && SEED), "the seed iteration gathers every source");
  uint64_t item = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  if (item >= n_items) return;  // whole warp exits together
  if (LISTED) item = item_list[item];   // sharded: n_items counts the owned items, listed ascending
  const uint32_t lane = threadIdx.x & 31, sub = lane & 3, q = lane >> 2;
  const uint32_t row = item_row[item];
  if (!owned_row(peers, row)) return;  // sharded: another rank owns this row (warp-uniform)
  const uint32_t chunk = (uint32_t)item - item_start[row - warp_row_begin];
  const uint32_t rs = row_ptr[row], re = row_ptr[row + 1];
  const uint32_t e0 = rs + chunk * (uint32_t)CHUNK_EDGES;
  const uint32_t e1 = min(e0 + (uint32_t)CHUNK_EDGES, re);
  uint4 acc = make_uint4(0, 0, 0, 0);
  // out-of-range lanes and (FRONTIER) unchanged sources are redirected to the row itself: merging one's own row
  // is a no-op under max, so the gather loop is branch-free
  uint32_t nxt = (e0 + lane < e1) ? ld_stream_u32(col + e0 + lane) : row;
  if (SEED) {
    // SEED (see quad_rows): each lane loads the 2-B seed of its source, one batch ahead, and the index one batch
    // further; each quad then takes four of the 32 seeds by shuffle and folds in their slices
    uint32_t sn = __ldg(seed + nxt);
    nxt = (e0 + 32 + lane < e1) ? ld_stream_u32(col + e0 + 32 + lane) : row;
    for (uint32_t base = e0; base < e1; base += 32) {
      const uint32_t mine = sn;
      sn = __ldg(seed + nxt);
      nxt = (base + 64 + lane < e1) ? ld_stream_u32(col + base + 64 + lane) : row;
      const uint32_t s0 = __shfl_sync(0xffffffffu, mine, q);
      const uint32_t s1 = __shfl_sync(0xffffffffu, mine, q + 8);
      const uint32_t s2 = __shfl_sync(0xffffffffu, mine, q + 16);
      const uint32_t s3 = __shfl_sync(0xffffffffu, mine, q + 24);
      acc = vmax_u8x16(vmax_u8x16(acc, seed_slice(s0, sub)),
                       vmax_u8x16(vmax_u8x16(seed_slice(s1, sub), seed_slice(s2, sub)), seed_slice(s3, sub)));
    }
  } else
  for (uint32_t base = e0; base < e1; base += 32) {
    uint32_t mine = nxt;
    nxt = (base + 32 + lane < e1) ? ld_stream_u32(col + base + 32 + lane) : row;
    if (FRONTIER) mine = bm_test(bm_prev, mine) ? mine : row;
    const uint32_t i0 = __shfl_sync(0xffffffffu, mine, q);
    const uint32_t i1 = __shfl_sync(0xffffffffu, mine, q + 8);
    const uint32_t i2 = __shfl_sync(0xffffffffu, mine, q + 16);
    const uint32_t i3 = __shfl_sync(0xffffffffu, mine, q + 24);
    const uint4 v0 = ld_gather_u4(oldr + (uint64_t)i0 * 4 + sub, i0 < l1_hub);
    const uint4 v1 = ld_gather_u4(oldr + (uint64_t)i1 * 4 + sub, i1 < l1_hub);
    const uint4 v2 = ld_gather_u4(oldr + (uint64_t)i2 * 4 + sub, i2 < l1_hub);
    const uint4 v3 = ld_gather_u4(oldr + (uint64_t)i3 * 4 + sub, i3 < l1_hub);
    acc = vmax_u8x16(vmax_u8x16(acc, v0), vmax_u8x16(vmax_u8x16(v1, v2), v3));
  }
#pragma unroll
  for (int off = 4; off < 32; off <<= 1) {
    uint4 o;
    o.x = __shfl_xor_sync(0xffffffffu, acc.x, off); o.y = __shfl_xor_sync(0xffffffffu, acc.y, off);
    o.z = __shfl_xor_sync(0xffffffffu, acc.z, off); o.w = __shfl_xor_sync(0xffffffffu, acc.w, off);
    acc = vmax_u8x16(acc, o);
  }
  if (item < first_multi_free_item) {  // this row spans several items: park the partial maximum
    if (q == 0) partial[item * 4 + sub] = acc;
    return;
  }
  const uint4 own = SEED ? seed_slice(__ldg(seed + row), sub)
                         : ld_gather_u4(oldr + (uint64_t)row * 4 + sub, row < l1_hub);
  acc = vmax_u8x16(acc, own);
  const unsigned ball = __ballot_sync(0xffffffffu, ne_u4(acc, own));
  const bool changed = (ball & 0xFu) != 0u;
  if (q == 0) publish_row(newr, bm_cur, peers, row, sub, acc, changed || bm_test(bm_prev, row), changed);
}

// rows spanning several work items: one warp reduces the parked partials (the own row comes from `oldr` in the seed
// iteration too: it equals the seed's row then, and these are a few rows)
__global__ void __launch_bounds__(256) k_pull_merge(uint64_t n_rows, const uint32_t* __restrict__ item_start,
    uint32_t warp_row_begin, const uint4* __restrict__ partial, const uint4* __restrict__ oldr,
    uint4* __restrict__ newr, const uint32_t* __restrict__ bm_prev, uint32_t* __restrict__ bm_cur, const PeerOut peers) {
  const uint64_t r = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  if (r >= n_rows) return;
  const uint32_t lane = threadIdx.x & 31, sub = lane & 3, q = lane >> 2;
  const uint32_t row = warp_row_begin + (uint32_t)r;
  if (!owned_row(peers, row)) return;
  const uint32_t i0 = item_start[r], i1 = item_start[r + 1];
  uint4 acc = make_uint4(0, 0, 0, 0);
  for (uint32_t it = i0 + q; it < i1; it += 8) acc = vmax_u8x16(acc, ld_stream_u4(partial + (uint64_t)it * 4 + sub));
#pragma unroll
  for (int off = 4; off < 32; off <<= 1) {
    uint4 o;
    o.x = __shfl_xor_sync(0xffffffffu, acc.x, off); o.y = __shfl_xor_sync(0xffffffffu, acc.y, off);
    o.z = __shfl_xor_sync(0xffffffffu, acc.z, off); o.w = __shfl_xor_sync(0xffffffffu, acc.w, off);
    acc = vmax_u8x16(acc, o);
  }
  const uint4 own = oldr[(uint64_t)row * 4 + sub];
  acc = vmax_u8x16(acc, own);
  const unsigned ball = __ballot_sync(0xffffffffu, ne_u4(acc, own));
  const bool changed = (ball & 0xFu) != 0u;
  if (q == 0) publish_row(newr, bm_cur, peers, row, sub, acc, changed || bm_test(bm_prev, row), changed);
}

// ---- push from a small frontier (update_changed_counters, harmonic.rs:75-114) --------------------------
// The push SOURCES are the frontier nodes (previous iteration's changed bitmap) with at least one out-edge, listed in node
// order; source j owns the push slots [off[j], off[j+1]), one per out-edge (of an owned destination, on a sharded handle).
// The list is built without atomics, so it is the same every run: per bitmap word, k_frontier_count packs
// (sources << 32 | out-edges); a CUB exclusive scan over the words gives every word its first source and first slot, and
// k_frontier_scatter writes the list.  The halves of the packed sum never carry into each other: the slot total is at most
// E < 2^32 (fwd_ptr is u32).  A frontier node without out-edges is not a source, so every source has >= 1 slot (k_push
// relies on it).
__global__ void k_frontier_count(const uint32_t* __restrict__ bm, uint64_t words, const uint32_t* __restrict__ fwd_ptr,
                                 unsigned long long* __restrict__ word_sum) {
  const uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (w > words) return;
  uint32_t m = w < words ? bm[w] : 0u;   // entry `words` is 0: its scanned value is the total
  uint32_t n = 0, d = 0;
  while (m) {
    const uint32_t v = (uint32_t)(w * 32 + (__ffs(m) - 1));
    m &= m - 1;
    const uint32_t dv = fwd_ptr[v + 1] - fwd_ptr[v];
    n += dv != 0u; d += dv;
  }
  word_sum[w] = ((unsigned long long)n << 32) | d;
}
// slot_total (sharded handles): the number of push slots of this rank, for the host
__global__ void k_frontier_scatter(const uint32_t* __restrict__ bm, uint64_t words, const uint32_t* __restrict__ fwd_ptr,
                                   const unsigned long long* __restrict__ word_pos, uint32_t* __restrict__ list,
                                   uint32_t* __restrict__ fbeg, uint32_t* __restrict__ off, unsigned long long* slot_total) {
  const uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (w > words) return;
  const unsigned long long p = word_pos[w];
  uint32_t j = (uint32_t)(p >> 32), o = (uint32_t)p;
  if (w == words) {   // off[n_sources] = slot total
    off[j] = o;
    if (slot_total) *slot_total = o;
    return;
  }
  uint32_t m = bm[w];
  while (m) {
    const uint32_t v = (uint32_t)(w * 32 + (__ffs(m) - 1));
    m &= m - 1;
    const uint32_t f0 = fwd_ptr[v], dv = fwd_ptr[v + 1] - f0;
    if (!dv) continue;
    list[j] = v; fbeg[j] = f0; off[j] = o;
    j++; o += dv;
  }
}
// refresh the two-iteration-old rows of the frontier nodes; one quad per bitmap word.  A sharded handle refreshes the rows
// it owns (whole bitmap words, see owned_row); the others arrive from their owners.
__global__ void k_copy_stale(const uint32_t* __restrict__ bm, uint64_t words, const uint4* __restrict__ oldr,
                             uint4* __restrict__ newr, uint32_t world, uint32_t rank) {
  const uint64_t gt = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const uint64_t w = (gt >> 2) * world + rank;   // this rank's k-th bitmap word
  if (w >= words) return;
  uint32_t m = __ldg(bm + w);
  while (m) {
    const uint64_t v = w * 32 + (uint64_t)(__ffs(m) - 1);
    m &= m - 1;
    newr[v * 4 + (gt & 3)] = oldr[v * 4 + (gt & 3)];
  }
}
// fused exchange after a push: every owned row that was refreshed or changed in this iteration goes to the peers
// (the frontier is small by construction: one quad per OWNED bitmap word, i.e. per 32-row block, walks the set bits)
__global__ void k_publish_rows(const uint32_t* __restrict__ bm_prev, const uint32_t* __restrict__ bm_cur, uint64_t n_rows,
                               const uint4* __restrict__ newr, const PeerOut peers) {
  const uint64_t gt = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const uint64_t w = (gt >> 2) * peers.world + peers.rank;     // this rank's k-th bitmap word
  if (w * 32 >= n_rows) return;
  uint32_t m = __ldg(bm_prev + w) | __ldg(bm_cur + w);
  while (m) {
    const uint64_t row = w * 32 + (uint64_t)(__ffs(m) - 1);
    m &= m - 1;
    if (row >= n_rows) break;
    const uint4 v = newr[row * 4 + (gt & 3)];
    const uint32_t want = peers.sub ? __ldg(peers.sub + row) : 0xFFFFFFFFu;
    for (int p = 0; p < peers.n; p++) if ((want >> peers.prank[p]) & 1u) peers.newr[p][row * 4 + (gt & 3)] = v;
  }
}
// Load-balanced push.  The slots are cut into one contiguous tile per warp (a multiple of 32 slots), so a source with many
// out-edges spreads over several warps and every warp gets the same work.  A warp finds the source of its first slot with
// one binary search over `off`, then walks its tile 32 slots at a time:
//   * the lanes load the window of sources cur .. cur+31 (list, fbeg, off: coalesced).  The 32 slots of a chunk lie in at
//     most 32 sources, because every source has >= 1 slot; each lane finds its slot's source by a 5-step search over the
//     shuffled window ends and loads its destination (consecutive slots of one source read consecutive fwd_dst words);
//   * each half-warp then takes every other slot: one 64-B row, 16 lanes x 4 B.  The source row stays in registers while
//     consecutive slots share the source; PUSH_BATCH destination rows are loaded and their first CAS issued before any
//     result is waited for, so several rows per half-warp are in flight.  The byte max is a 32-bit CAS loop (bmax4_7bit);
//     a destination that changed gets its bit in bm_cur.
// `total` = the scanned (sources << 32 | slots) of the whole frontier (the last entry of the scan): the source count is
// known only on the device.
constexpr int PUSH_BATCH = 4;
constexpr int PUSH_CTAS_PER_SM = 6;   // 40 registers without spills
__global__ void __launch_bounds__(256, PUSH_CTAS_PER_SM) k_push(const unsigned long long* __restrict__ total, const uint32_t* __restrict__ list,
    const uint32_t* __restrict__ fbeg, const uint32_t* __restrict__ off, const uint32_t* __restrict__ fwd_dst,
    const uint32_t* __restrict__ old32, uint32_t* new32, uint32_t* __restrict__ bm_cur) {
  const unsigned long long tot = *total;
  const uint32_t n_src = (uint32_t)(tot >> 32), n_slots = (uint32_t)tot;
  const uint32_t lane = threadIdx.x & 31, l = lane & 15, half = lane >> 4;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  const uint64_t warp = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  const uint64_t tile = ((n_slots + n_warps - 1) / n_warps + 31) & ~31ull;
  if (warp * tile >= n_slots) return;   // whole warp
  const uint32_t s0 = (uint32_t)(warp * tile), s1 = (uint32_t)min(warp * tile + tile, (uint64_t)n_slots);
  uint32_t lo = 0, hi = n_src;   // cur = last source j with off[j] <= s0
  while (lo + 1 < hi) { const uint32_t mid = (lo + hi) >> 1; if (off[mid] <= s0) lo = mid; else hi = mid; }
  uint32_t cur = lo;
  uint32_t row_u = 0xFFFFFFFFu, row = 0;   // this half-warp's source row
  for (uint32_t S = s0; S < s1; S += 32) {
    const uint32_t wj = min(cur + lane, n_src - 1);
    const uint32_t w_end = off[min(cur + lane + 1, n_src)];   // end of source cur+lane (the slot total past the last one)
    const uint32_t w_beg = off[wj], w_u = list[wj], w_f = fbeg[wj];
    const uint32_t s = S + lane;
    uint32_t k = 0;   // number of window sources that end at or before slot s: its source is cur + k (k <= 31)
#pragma unroll
    for (uint32_t step = 16; step; step >>= 1) {
      const uint32_t e = __shfl_sync(0xffffffffu, w_end, k + step - 1);
      if (e <= s) k += step;
    }
    const uint32_t u = __shfl_sync(0xffffffffu, w_u, k);
    const uint32_t e_first = __shfl_sync(0xffffffffu, w_f, k) + (s - __shfl_sync(0xffffffffu, w_beg, k));
    const uint32_t n_here = min(32u, s1 - S);
    const uint32_t v = lane < n_here ? ld_stream_u32(fwd_dst + e_first) : 0u;
    cur += __popc(__ballot_sync(0xffffffffu, w_end <= S + 32));   // source of slot S + 32
    for (uint32_t p0 = 0; p0 < n_here; p0 += 2 * PUSH_BATCH) {
      uint32_t dst[PUSH_BATCH], mine[PUSH_BATCH], old[PUSH_BATCH], want[PUSH_BATCH], got[PUSH_BATCH];
      bool live[PUSH_BATCH];
#pragma unroll
      for (int q = 0; q < PUSH_BATCH; q++) {
        const uint32_t from = p0 + 2 * q + half;   // lane holding this half-warp's q-th slot
        const uint32_t uq = __shfl_sync(0xffffffffu, u, from);
        dst[q] = __shfl_sync(0xffffffffu, v, from);
        live[q] = from < n_here;
        if (live[q] && uq != row_u) { row = __ldg(old32 + (uint64_t)uq * 16 + l); row_u = uq; }
        mine[q] = row;
      }
#pragma unroll
      for (int q = 0; q < PUSH_BATCH; q++) old[q] = live[q] ? new32[(uint64_t)dst[q] * 16 + l] : 0u;
#pragma unroll
      for (int q = 0; q < PUSH_BATCH; q++) {
        want[q] = live[q] ? bmax4_7bit(old[q], mine[q]) : old[q];
        got[q] = want[q] != old[q] ? atomicCAS(new32 + (uint64_t)dst[q] * 16 + l, old[q], want[q]) : old[q];
      }
#pragma unroll
      for (int q = 0; q < PUSH_BATCH; q++) {
        bool changed = want[q] != old[q] && got[q] == old[q];
        if (want[q] != old[q] && !changed) {   // another push got there first: retry against its value
          uint32_t* addr = new32 + (uint64_t)dst[q] * 16 + l;
          uint32_t c = got[q], m = bmax4_7bit(c, mine[q]);
          while (m != c) {
            const uint32_t prev = atomicCAS(addr, c, m);
            if (prev == c) { changed = true; break; }
            c = prev; m = bmax4_7bit(c, mine[q]);
          }
        }
        const unsigned ball = __ballot_sync(0xffffffffu, changed);
        if (((ball >> (16 * half)) & 0xFFFFu) && l == 0) atomicOr(bm_cur + (dst[q] >> 5), 1u << (dst[q] & 31));
      }
    }
  }
}

// ---- centrality update for the nodes touched this iteration -------------------------------------------
__global__ void __launch_bounds__(256) k_finalize(uint64_t row_begin, uint64_t row_end,
    const uint4* __restrict__ newr, const uint32_t* __restrict__ bm_prev, const uint32_t* __restrict__ bm_cur,
    uint64_t* __restrict__ size_cache, double* __restrict__ ksum, double* __restrict__ kerr,
    const uint32_t* __restrict__ fwd_ptr, double t_plus_1, unsigned long long* counters, const uint32_t own_world,
    const uint32_t own_rank) {
  __shared__ HllTables tab;
  __shared__ unsigned long long s_cnt[2];
  for (int i = threadIdx.x; i < (int)(sizeof(HllTables) / 8); i += blockDim.x) ((double*)&tab)[i] = ((const double*)&c_tab)[i];
  if (threadIdx.x < 2) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  // persistent grid: the tables are staged once per CTA, each warp then walks whole 32-row blocks -- only the blocks this
  // rank owns, and only those with a bit set in either bitmap word (late iterations touch a few thousand rows)
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t world = own_world > 1 ? own_world : 1;
  const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5), w0 = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const uint64_t b0 = row_begin >> 5, b1 = (row_end + 31) >> 5;
  const uint64_t first = b0 + ((uint64_t)own_rank + world - b0 % world) % world;
  unsigned long long my_changed = 0, my_out = 0;
  for (uint64_t b = first + w0 * world; b < b1; b += warps * world) {
    const uint32_t wc = __ldg(bm_cur + b), wp = __ldg(bm_prev + b);
    if ((wc | wp) == 0u) continue;
    const uint64_t v = b * 32 + lane;
    const bool bc = (wc >> lane) & 1u, bp = (wp >> lane) & 1u;
    if (v >= row_begin && v < row_end && (bc || bp)) {
      double s = ksum[v], e = kerr[v];
      if (bc) {
        uint32_t w[16];
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const uint4 x = newr[v * 4 + q];
          w[4 * q] = x.x; w[4 * q + 1] = x.y; w[4 * q + 2] = x.z; w[4 * q + 3] = x.w;
        }
        const uint64_t sn = hll64_size(w, &tab);
        const uint64_t so = size_cache[v];
        const uint64_t d = sn >= so ? sn - so : 0ull;  // checked_sub().unwrap_or_default()
        kahan_add(s, e, __ddiv_rn(__ull2double_rn(d), t_plus_1));
        size_cache[v] = sn;
        my_changed += 1;
        if (fwd_ptr) my_out += fwd_ptr[v + 1] - fwd_ptr[v];
      } else {
        kahan_add(s, e, 0.0);  // the reference adds 0/(t+1) to every unchanged node; once is enough
      }
      ksum[v] = s; kerr[v] = e;
    }
  }
  // block reduce the two counters
  for (int off = 16; off; off >>= 1) {
    my_changed += __shfl_down_sync(0xffffffffu, my_changed, off);
    my_out += __shfl_down_sync(0xffffffffu, my_out, off);
  }
  if ((threadIdx.x & 31) == 0 && (my_changed | my_out)) { atomicAdd(&s_cnt[0], my_changed); atomicAdd(&s_cnt[1], my_out); }
  __syncthreads();
  if (threadIdx.x == 0 && (s_cnt[0] | s_cnt[1])) { atomicAdd(counters + 0, s_cnt[0]); atomicAdd(counters + 1, s_cnt[1]); }
}

// ---- result / debug gathers ------------------------------------------------------------------------------
__global__ void k_result_flags(const uint32_t* __restrict__ inv, const double* __restrict__ ksum, uint64_t N,
                               uint64_t row_begin, uint64_t row_end, double norm, uint32_t* flag, double* val,
                               const uint32_t own_world, const uint32_t own_rank) {
  uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (r >= N) return;
  const uint32_t v = inv[r];
  double c = ksum[v];
  const bool keep = (c > 0.0) && v >= row_begin && v < row_end &&  // normalize_centralities harmonic.rs:178-195
                    (own_world <= 1 || ((v >> 5) % own_world) == own_rank);
  c = __ddiv_rn(c, norm);
  if (isinf(c) || isnan(c)) c = 0.0;
  flag[r] = keep ? 1u : 0u;
  val[r] = c;
}
__global__ void k_result_scatter(const uint32_t* __restrict__ flag, const uint32_t* __restrict__ pos,
                                 const double* __restrict__ val, const uint64_t* __restrict__ id_lo,
                                 const uint64_t* __restrict__ id_hi, uint64_t N, uint64_t cap, uint64_t* out_lo,
                                 uint64_t* out_hi, double* out_c) {
  uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (r >= N || !flag[r]) return;
  uint32_t p = pos[r];
  if (p >= cap) return;
  out_lo[p] = id_lo[r]; out_hi[p] = id_hi[r]; out_c[p] = val[r];
}
__global__ void k_gather_regs(const uint32_t* __restrict__ inv, const uint4* __restrict__ regs, uint64_t first,
                              uint64_t count, uint4* out) {
  uint64_t gt = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  uint64_t i = gt >> 2;
  if (i >= count) return;
  out[i * 4 + (gt & 3)] = regs[(uint64_t)inv[first + i] * 4 + (gt & 3)];
}
__global__ void k_gather_f64x2(const uint32_t* __restrict__ inv, const double* __restrict__ a, const double* __restrict__ b,
                               uint64_t first, uint64_t count, double* oa, double* ob) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= count) return;
  uint32_t v = inv[first + i];
  oa[i] = a[v]; ob[i] = b[v];
}

// Rows are ordered by in-degree, so the head of the register array holds the hubs -- on a power-law graph also the
// most-gathered sources.  The first L2_WINDOW_BYTES of the array being READ are pinned as persisting L2 lines for the pull
// kernels (stream access-policy window, re-pointed at the `old` array every iteration), so the streaming col/row traffic
// cannot evict them.
// H100 80 GB at 400 W, C2 (25 M ids / 500 M edges): 0 -> 53.6, 16 -> 47.9, 32 -> 67.0 ms/step (32 of the 50 MB L2 starve the streams)
// The seed iteration (t = 0) points the window at the seed array instead, capped at the same size.  Iteration 0 of C2
// (28.8 MB of seeds), same card: no window 6.87, 16 MB 6.93, the whole array (a 30 MB window) 6.18 ms -- but a
// 30 MB set-aside slows the dense iterations from 8.4 to 10.3 ms, so the cap stays.
// Re-timed with tools/dense_iter_sweep.py (H100 80 GB at 700 W, ms per computation): 16 MB 39.11, 20 MB 39.00, 24 MB 39.60 --
// 20 MB is inside the spread of 16 MB, so 16 MB stays.  Evict-first L2 hints on the pulls' read-once traffic (col, row_ptr,
// own rows, new-row stores) changed none of these by more than the spread (DESIGN section 6), so the pulls carry none.
constexpr uint64_t L2_WINDOW_BYTES = 16ull << 20;
constexpr uint64_t SEED_WINDOW_BYTES = 16ull << 20;   // the cap of the seed iteration's window, whatever the pulls' window

// The pulls keep their hub sources in L1 (ld_gather_u4).  None of them uses shared memory, so they prefer the largest L1
// carve-out: the hubs are then not limited by a carve-out the driver picked.
static int pulls_prefer_l1() {
#ifndef SB200_EMU
  const void* pulls[] = {
      (const void*)k_pull_quad<false, false>, (const void*)k_pull_quad<true, false>, (const void*)k_pull_quad<false, true>,
      (const void*)k_pull_quad_owned<false, false>, (const void*)k_pull_quad_owned<true, false>,
      (const void*)k_pull_quad_owned<false, true>,
      (const void*)k_pull_warp<false, false, false>, (const void*)k_pull_warp<true, false, false>,
      (const void*)k_pull_warp<false, false, true>, (const void*)k_pull_warp<false, true, false>,
      (const void*)k_pull_warp<true, true, false>, (const void*)k_pull_warp<false, true, true>,
      (const void*)k_pull_merge};
  for (const void* k : pulls)
    SB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxL1));
#endif
  return SB200_OK;
}

int hb_set_l2_window(sb200_graph* g, uint64_t want);
int hb_alloc_state(sb200_graph* g) {
  const uint64_t N = g->N;
  const uint64_t words = (N + 31) / 32;
  SB_TRY(load_tables(g->device));
  SB_TRY(g->regs[0].alloc(std::max<uint64_t>(N, 1) * 64));
  SB_TRY(g->regs[1].alloc(std::max<uint64_t>(N, 1) * 64));
  SB_TRY(g->seed.alloc(std::max<uint64_t>(N, 1)));
  SB_TRY(g->bm[0].alloc(words + 1)); SB_TRY(g->bm[1].alloc(words + 1));
  SB_TRY(g->size_cache.alloc(std::max<uint64_t>(N, 1)));
  SB_TRY(g->kahan_sum.alloc(std::max<uint64_t>(N, 1))); SB_TRY(g->kahan_err.alloc(std::max<uint64_t>(N, 1)));
  SB_TRY(g->counters.alloc(8));
  if (g->world > 1) {   // sync page of the device-side barrier (plain cudaMalloc: exported through CUDA IPC)
    SB_TRY(g->sync_page.alloc(SYNC_SLOTS));
    SB_CUDA(cudaMemset(g->sync_page.p, 0, SYNC_SLOTS * sizeof(unsigned long long)));
  }
  if (!g->h_counters) SB_CUDA(cudaMallocHost((void**)&g->h_counters, 8 * sizeof(unsigned long long)));
  return hb_set_l2_window(g, L2_WINDOW_BYTES);
}

static int set_l2_window(cudaStream_t s, const void* base, uint64_t bytes);
// the persisting window of the pulls: `want` bytes, capped by the device and the register array (0: no window).  The caller
// has made g->device current.
int hb_set_l2_window(sb200_graph* g, uint64_t want) {
  cudaDeviceProp prop;
  SB_CUDA(cudaGetDeviceProperties(&prop, g->device));
  want = std::min<uint64_t>(want, (uint64_t)std::max(prop.persistingL2CacheMaxSize, 0));
  want = std::min<uint64_t>(want, (uint64_t)std::max(prop.accessPolicyMaxWindowSize, 0));
  want = std::min<uint64_t>(want, g->N * 64);
  const bool had = g->l2_window_bytes != 0;
  g->l2_window_bytes = 0;
  if (want) { SB_CUDA(cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want)); g->l2_window_bytes = want; return SB200_OK; }
  if (had) {
    // no window any more: the pulls stop re-pointing one (hb_step_launch), so drop the one the last pull left on each stream,
    // give the set-aside back and turn the lines already pinned into normal ones
    SB_TRY(set_l2_window(g->stream, nullptr, 0));
    if (g->side_stream) SB_TRY(set_l2_window(g->side_stream, nullptr, 0));
    SB_CUDA(cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, 0));
    SB_CUDA(cudaCtxResetPersistingL2Cache());
  }
  return SB200_OK;
}

int hb_reset(sb200_graph* g) {
  cudaStream_t s = g->stream;
  const uint64_t N = g->N, words = (N + 31) / 32;
  g->cur = 0; g->bcur = 0; g->t = 0; g->has_changes = N > 0; g->exchange_pending = false;
  g->n_changed_prev = N; g->frontier_edges_prev = g->E_kept;
  if (N == 0) return SB200_OK;
  SB_LAUNCH(k_hb_init, div_up(N * 4, 256), 256, 0, s, g->id_lo.p, g->perm.p, N, (uint4*)g->regs[0].p, (uint4*)g->regs[1].p,
            g->seed.p, g->size_cache.p, g->kahan_sum.p, g->kahan_err.p);
  SB_CHECK_LAUNCH();
  SB_LAUNCH(k_bm_fill, div_up(words, 256), 256, 0, s, g->bm[0].p, N, words);  // changed_nodes filled, harmonic.rs:223-225
  SB_CHECK_LAUNCH();
  SB_CUDA(cudaMemsetAsync(g->bm[1].p, 0, (words + 1) * 4, s));
  SB_CUDA(cudaStreamSynchronize(s));
  return SB200_OK;
}

#define PROF_BEGIN(g, fam) do { if ((g)->profiling) { SB_CUDA(cudaEventRecord((g)->prof_ev[fam][0], (g)->stream)); } } while (0)
#define PROF_END(g, fam, bytes) do { if ((g)->profiling) { SB_CUDA(cudaEventRecord((g)->prof_ev[fam][1], (g)->stream)); \
    (g)->prof_used[fam] = true; (g)->prof_step_bytes[fam] = (double)(bytes); } } while (0)

// publish targets of the iteration being launched: the peers' copies of the `new` register array / `cur` bitmap
static PeerOut make_peer_out(const sb200_graph* g, bool with_targets) {
  PeerOut po;
  memset(&po, 0, sizeof(po));
  po.world = (uint32_t)g->world; po.rank = (uint32_t)g->rank;
  if (with_targets && g->p2p) {
    po.n = g->n_peers;
    po.sub = (g->publish_all || !g->sub_mask.p) ? nullptr : g->sub_mask.p;
    for (int p = 0; p < g->n_peers; p++) {
      po.newr[p] = (uint4*)g->peer_regs[g->cur ^ 1][p]; po.bmc[p] = (uint32_t*)g->peer_bm[g->bcur ^ 1][p];
      po.prank[p] = (uint8_t)g->peer_rank[p];
    }
  }
  return po;
}

// persisting-L2 access-policy window of the pull kernels on stream `s` (see hb_alloc_state); 0 bytes: none
static int set_l2_window(cudaStream_t s, const void* base, uint64_t bytes) {
  cudaStreamAttrValue a;
  memset(&a, 0, sizeof(a));
  a.accessPolicyWindow.base_ptr = (void*)base; a.accessPolicyWindow.num_bytes = bytes;
  a.accessPolicyWindow.hitRatio = 1.0f; a.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
  a.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
  SB_CUDA(cudaStreamSetAttribute(s, cudaStreamAttributeAccessPolicyWindow, &a));
  return SB200_OK;
}
// the window of a pull: the head of the `old` array, or in the seed iteration the head of the seed array
static void l2_window_of(const sb200_graph* g, const uint4* oldr, bool from_seed, const void** base, uint64_t* bytes) {
  *base = from_seed ? (const void*)g->seed.p : (const void*)oldr;
  *bytes = from_seed ? std::min<uint64_t>(std::min<uint64_t>(g->l2_window_bytes, SEED_WINDOW_BYTES), g->N * sizeof(uint16_t))
                     : g->l2_window_bytes;
}

template <bool FRONTIER, bool SEED>
static int launch_pull(sb200_graph* g, const uint4* oldr, uint4* newr, const uint32_t* bmp, uint32_t* bmc) {
  cudaStream_t s = g->stream;
  const PeerOut po = make_peer_out(g, true);
  const int FW = SEED ? sb200_graph::F_PULL_WARP_SEED : FRONTIER ? sb200_graph::F_PULL_WARP_FRONT : sb200_graph::F_PULL_WARP_DENSE;
  const int FQ = SEED ? sb200_graph::F_PULL_QUAD_SEED : FRONTIER ? sb200_graph::F_PULL_QUAD_FRONT : sb200_graph::F_PULL_QUAD_DENSE;
  // per edge: the col index, + the 64-B gather when every source is read, or + its 2-B seed in the seed iteration
  const double per_edge = SEED ? 6.0 : FRONTIER ? 4.0 : 68.0;
  // fused exchange: short rows on the side stream, next to the long-row kernel (see k_pull_quad_owned)
  if (g->opt_side_ctas < 0) {
    // default: the side stream for up to 4 ranks and for one multicast target; with unicast stores to 7 peers the short-row
    // kernel beside the long-row one slows both (not measured on H100: it needs several GPUs; set_option("quad_side_ctas")
    // overrides)
    const bool multicast_target = g->n_peers < g->world - 1;
    g->opt_side_ctas = (multicast_target || g->world <= 4) ? 2 : 0;
  }
  const int side_ctas = g->opt_side_ctas;
  const uint32_t l1_hub = (uint32_t)std::min<uint64_t>(g->l1_hub_bytes / 64, g->N);
  const bool side_quad = side_ctas > 0 && g->world > 1 && g->p2p && g->n_peers > 0 && g->n_items && g->quad_row_end > g->quad_row_begin;
  if (side_quad) {
    if (!g->side_stream) {
      int lo = 0, hi = 0;
      SB_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
      SB_CUDA(cudaStreamCreateWithPriority(&g->side_stream, cudaStreamNonBlocking, hi));
      SB_CUDA(cudaEventCreateWithFlags(&g->ev_fork, cudaEventDisableTiming));
      SB_CUDA(cudaEventCreateWithFlags(&g->ev_join, cudaEventDisableTiming));
      SB_CUDA(cudaEventCreate(&g->side_prof[0])); SB_CUDA(cudaEventCreate(&g->side_prof[1]));
    }
    if (!g->sm_count) SB_CUDA(cudaDeviceGetAttribute(&g->sm_count, cudaDevAttrMultiProcessorCount, g->device));
    const int sm_count = g->sm_count;
    const uint64_t world = (uint64_t)g->world, b0 = g->quad_row_begin >> 5, b1 = (g->quad_row_end - 1) >> 5;
    const uint64_t first = b0 + ((uint64_t)g->rank + world - b0 % world) % world;
    const uint64_t n_tasks = first <= b1 ? ((b1 - first) / world + 1) * 4 : 0;
    SB_CUDA(cudaEventRecord(g->ev_fork, s));
    SB_CUDA(cudaStreamWaitEvent(g->side_stream, g->ev_fork, 0));
    if (g->l2_window_bytes) {
      const void* wbase; uint64_t wbytes;
      l2_window_of(g, oldr, SEED, &wbase, &wbytes);
      SB_TRY(set_l2_window(g->side_stream, wbase, wbytes));
    }
    if (g->profiling) SB_CUDA(cudaEventRecord(g->side_prof[0], g->side_stream));
    if (n_tasks) {
      const unsigned grid = (unsigned)std::min<uint64_t>(div_up(n_tasks, 8), (uint64_t)sm_count * (uint64_t)side_ctas);
      auto kern = k_pull_quad_owned<FRONTIER, SEED>;
      SB_LAUNCH(kern, grid, 256, 0, g->side_stream, g->quad_row_begin, g->quad_row_end, first, n_tasks,
                g->row_ptr.p, g->col.p, oldr, g->seed.p, newr, bmp, bmc, po, l1_hub);
      SB_CHECK_LAUNCH();
    }
    if (g->profiling) {
      SB_CUDA(cudaEventRecord(g->side_prof[1], g->side_stream));
      g->side_prof_used = true; g->side_prof_family = FQ;
      g->prof_step_bytes[FQ] = g->own_frac * (per_edge * (double)g->E_quad + 68.0 * (double)(g->quad_row_end - g->quad_row_begin));
    }
  }
  if (g->n_items) {
    PROF_BEGIN(g, FW);
    const bool listed = g->opt_owned_list > 0 && g->world > 1 && g->owned_items.p;
    const uint64_t n_launch = listed ? g->n_owned_items : g->n_items;
    auto kern = listed ? k_pull_warp<FRONTIER, true, SEED> : k_pull_warp<FRONTIER, false, SEED>;
    if (n_launch)
    SB_LAUNCH(kern, div_up(n_launch * 32, 256), 256, 0, s, n_launch, g->n_multi_items,
              listed ? g->owned_items.p : (const uint32_t*)nullptr, g->item_row.p, g->item_start.p, (uint32_t)g->warp_row_begin, g->row_ptr.p, g->col.p, oldr,
              g->seed.p, newr, g->partial.p, bmp, bmc, po, l1_hub);
    SB_CHECK_LAUNCH();
    PROF_END(g, FW, g->own_frac * (per_edge * (double)g->E_warp + 68.0 * (double)(g->warp_row_end - g->warp_row_begin - g->n_multi_rows)));
  }
  if (g->n_multi_rows) {
    PROF_BEGIN(g, sb200_graph::F_PULL_MERGE);
    SB_LAUNCH(k_pull_merge, div_up(g->n_multi_rows * 32, 256), 256, 0, s, g->n_multi_rows, g->item_start.p,
              (uint32_t)g->warp_row_begin, g->partial.p, oldr, newr, bmp, bmc, po);
    SB_CHECK_LAUNCH();
    PROF_END(g, sb200_graph::F_PULL_MERGE, 64.0 * (double)g->n_multi_items + 68.0 * (double)g->n_multi_rows);
  }
  const uint64_t nq = g->quad_row_end - g->quad_row_begin;
  if (side_quad) { SB_CUDA(cudaEventRecord(g->ev_join, g->side_stream)); SB_CUDA(cudaStreamWaitEvent(s, g->ev_join, 0)); }
  else if (nq) {
    PROF_BEGIN(g, FQ);
    auto kern = k_pull_quad<FRONTIER, SEED>;
    SB_LAUNCH(kern, div_up(nq * 4, 256), 256, 0, s, g->quad_row_begin, g->quad_row_end, g->row_ptr.p,
              g->col.p, oldr, g->seed.p, newr, bmp, bmc, po, l1_hub);
    SB_CHECK_LAUNCH();
    PROF_END(g, FQ, g->own_frac * (per_edge * (double)g->E_quad + 68.0 * (double)nq));
  }
  return SB200_OK;
}

static int run_push(sb200_graph* g, const uint4* oldr, uint4* newr, const uint32_t* bmp, uint32_t* bmc) {
  cudaStream_t s = g->stream;
  const uint64_t N = g->N, words = (N + 31) / 32;
  const uint64_t nf = g->n_changed_prev;
  if (nf == 0) return SB200_OK;  // empty frontier: a converged state is a fixed point
  // the frontier's node count bounds the number of sources
  if (g->frontier_list.n < 2 * (nf + 1)) { SB_TRY(g->frontier_list.alloc(2 * (nf + 1) + (nf >> 1))); }
  if (g->frontier_off.n < nf + 1) { SB_TRY(g->frontier_off.alloc(nf + 1 + (nf >> 2))); }
  if (g->frontier_scan.n < 2 * (words + 1)) { SB_TRY(g->frontier_scan.alloc(2 * (words + 1))); }
  uint32_t* list = g->frontier_list.p;
  uint32_t* fbeg = g->frontier_list.p + g->frontier_list.n / 2;
  unsigned long long* word_sum = g->frontier_scan.p;
  unsigned long long* word_pos = g->frontier_scan.p + (words + 1);
  SB_LAUNCH(k_frontier_count, div_up(words + 1, 256), 256, 0, s, bmp, words, g->fwd_ptr.p, word_sum);
  SB_CHECK_LAUNCH();
  size_t need = 0;
  SB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, need, word_sum, word_pos, (int64_t)(words + 1), s));
  if (g->cub_tmp.n < need) SB_TRY(g->cub_tmp.alloc(need + 256));
  SB_CUDA(cub::DeviceScan::ExclusiveSum(g->cub_tmp.p, need, word_sum, word_pos, (int64_t)(words + 1), s));
  g_launches.fetch_add(2, std::memory_order_relaxed);
  SB_LAUNCH(k_frontier_scatter, div_up(words + 1, 256), 256, 0, s, bmp, words, g->fwd_ptr.p, word_pos, list, fbeg,
            g->frontier_off.p, g->world > 1 ? g->counters.p + 3 : (unsigned long long*)nullptr);
  SB_CHECK_LAUNCH();
  SB_LAUNCH(k_copy_stale, div_up(div_up(words, (uint64_t)g->world) * 4, 256), 256, 0, s, bmp, words, oldr, newr,
            (uint32_t)g->world, (uint32_t)g->rank);
  SB_CHECK_LAUNCH();
  uint64_t slots = g->frontier_edges_prev;
  if (g->world > 1) {   // this rank's share of the frontier's out-edges is not known from the previous step
    unsigned long long h = 0;
    SB_CUDA(cudaMemcpyAsync(&h, g->counters.p + 3, sizeof(h), cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaStreamSynchronize(s));
    slots = h;
  }
  if (slots) {
    // one wave of resident CTAs, and at least 32 slots per warp
    if (!g->sm_count) SB_CUDA(cudaDeviceGetAttribute(&g->sm_count, cudaDevAttrMultiProcessorCount, g->device));
    const unsigned grid = (unsigned)std::min<uint64_t>(div_up(slots, 32 * 8), (uint64_t)g->sm_count * PUSH_CTAS_PER_SM);
    PROF_BEGIN(g, sb200_graph::F_PUSH);
    SB_LAUNCH(k_push, grid, 256, 0, s, word_pos + words, list, fbeg, g->frontier_off.p, g->fwd_dst.p,
              (const uint32_t*)oldr, (uint32_t*)newr, bmc);
    SB_CHECK_LAUNCH();
    PROF_END(g, sb200_graph::F_PUSH, 132.0 * (double)slots);
  }
  if (g->p2p && g->n_peers > 0) {
    const PeerOut po = make_peer_out(g, true);
    SB_LAUNCH(k_publish_rows, div_up(div_up(words, (uint64_t)g->world) * 4, 256), 256, 0, s, bmp, bmc, N, (const uint4*)newr, po);
    SB_CHECK_LAUNCH();
  }
  return SB200_OK;
}

// fused exchange: each rank owns whole 32-row blocks, i.e. whole bitmap words; publish the owned words to the peers
__global__ void k_publish_bitmap(const uint32_t* __restrict__ bmc, uint64_t words, const PeerOut peers) {
  const uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (w >= words || (w % peers.world) != peers.rank) return;
  const uint32_t v = bmc[w];
  for (int p = 0; p < peers.n; p++) peers.bmc[p][w] = v;
}

// out-edges of the nodes in a changed bitmap (needed once, right after the lazy source-major CSR build)
__global__ void k_frontier_out_edges(const uint32_t* __restrict__ bm, uint64_t words, const uint32_t* __restrict__ fwd_ptr,
                                     unsigned long long* counter) {
  const uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  unsigned long long acc = 0;
  if (w < words) {
    uint32_t m = bm[w];
    while (m) { const int b = __ffs(m) - 1; m &= m - 1; const uint64_t v = w * 32 + b; acc += fwd_ptr[v + 1] - fwd_ptr[v]; }
  }
  for (int o = 16; o; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0 && acc) atomicAdd(counter, acc);
}

// ---- device-side barrier + changed-count sum across the ranks of one box ------------------------------------------------
// One warp.  Lane p stores (epoch, count) into slot [epoch & 1][my rank] of peer p's sync page (release, system scope,
// after a system fence that orders this rank's earlier peer stores -- the rows and bitmap words of the iteration --
// before the flag); lane r then spins (acquire) on slot [epoch & 1][r] of the LOCAL page until rank r's flag of this
// epoch has arrived, and the warp sums the counts.  Two parities: a rank can be at most one barrier ahead of the
// slowest one, so the slot of epoch e is rewritten (epoch e + 2) only after everybody has left barrier e + 1, i.e. has
// long read it.  A watchdog (globaltimer) turns a missing peer into an error instead of a hung GPU.
__device__ __forceinline__ void st_release_sys_u64(unsigned long long* p, unsigned long long v) {
#ifndef SB200_EMU
  asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
#else
  *(volatile unsigned long long*)p = v;
#endif
}
__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
#ifndef SB200_EMU
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
#else
  return *(const volatile unsigned long long*)p;
#endif
}
__device__ __forceinline__ unsigned long long global_ns() {
#ifndef SB200_EMU
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
#else
  return 0ull;
#endif
}
constexpr unsigned long long SYNC_COUNT_MASK = (1ull << 40) - 1;
__global__ void __launch_bounds__(32) k_barrier_count(const SyncView sv, unsigned long long epoch, const unsigned long long* __restrict__ count_in,
                                                      unsigned long long* out /* [0] total, [1] timed-out ranks */, unsigned long long timeout_ns) {
  const int lane = threadIdx.x;
  const unsigned long long e24 = epoch & 0xFFFFFFull;
  const unsigned long long cnt = count_in ? (*count_in & SYNC_COUNT_MASK) : 0ull;
  const unsigned long long val = (e24 << 40) | cnt;
  const uint32_t slot = (uint32_t)(epoch & 1ull) * 64u + sv.rank;
  __threadfence_system();
  if (lane < sv.n) st_release_sys_u64(sv.peer[lane] + slot, val);
  if (lane == sv.n) st_release_sys_u64(sv.local + slot, val);
  unsigned long long got = 0;
  bool ok = true;
  if (lane < (int)sv.world) {
    const unsigned long long* p = sv.local + (uint32_t)(epoch & 1ull) * 64u + lane;
    const unsigned long long t0 = global_ns();
    for (;;) {
      got = ld_acquire_sys_u64(p);
      if ((got >> 40) == e24) break;
      if (global_ns() - t0 > timeout_ns) { ok = false; got = 0; break; }
#ifdef SB200_EMU
      ok = false; got = 0; break;  // the emulator runs one rank at a time: a peer's flag cannot arrive while we wait
#endif
    }
  }
  unsigned long long sum = (lane < (int)sv.world && ok) ? (got & SYNC_COUNT_MASK) : 0ull;
  for (int o = 16; o; o >>= 1) sum += __shfl_down_sync(0xffffffffu, sum, o);
  const unsigned bad = __ballot_sync(0xffffffffu, !ok);
  if (lane == 0) { out[0] = sum; out[1] = (unsigned long long)__popc(bad); }
}

static SyncView make_sync_view(const sb200_graph* g) {
  SyncView sv;
  memset(&sv, 0, sizeof(sv));
  sv.local = g->sync_page.p; sv.n = g->n_peers; sv.world = (uint32_t)g->world; sv.rank = (uint32_t)g->rank;
  for (int p = 0; p < g->n_peers; p++) sv.peer[p] = (unsigned long long*)g->peer_sync[p];
  return sv;
}
// stand-alone barrier (before the first step of a run: every replica must be initialised before a peer may write into it)
int hb_barrier(sb200_graph* g) {
  cudaStream_t s = g->stream;
  if (!g->sync_page.p || g->n_peers != g->world - 1) SB_FAIL(SB200_ESTATE, "device barrier needs the sync pages of all %d peers", g->world - 1);
  for (int p = 0; p < g->n_peers; p++) if (!g->peer_sync[p]) SB_FAIL(SB200_ESTATE, "peer %d exported no sync page", p);
  g->sync_epoch++;
  SB_LAUNCH(k_barrier_count, 1, 32, 0, s, make_sync_view(g), (unsigned long long)g->sync_epoch, (const unsigned long long*)nullptr,
            g->counters.p + 5, 20000000000ull);
  SB_CHECK_LAUNCH();
  SB_CUDA(cudaMemcpyAsync(g->h_counters + 5, g->counters.p + 5, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  SB_CUDA(cudaStreamSynchronize(s));
  if (g->h_counters[6]) SB_FAIL(SB200_ESTATE, "inter-rank barrier timed out: %llu rank(s) did not arrive", (unsigned long long)g->h_counters[6]);
  return SB200_OK;
}

// One iteration = launch (everything queued on the handle's stream, nothing waited for) + finish (wait, read the
// counters, flip the ping-pong).  hb_step does both; the group / sharded run loops launch all ranks before they wait.
// with_barrier: the changed counts are summed across the ranks on the device (k_barrier_count) and the step finishes
// with the global count already applied (no sb200_hyperball_exchange_done needed).
int hb_step_launch(sb200_graph* g, bool with_barrier) {
  NvtxRange nvtx("sb200 hyperball iteration (launch)");
  cudaStream_t s = g->stream;
  const uint64_t N = g->N, words = (N + 31) / 32;
  if (g->step_in_flight) SB_FAIL(SB200_ESTATE, "the previous step has not been finished");
  if (g->exchange_pending) SB_FAIL(SB200_ESTATE, "sb200_hyperball_exchange_done() must be called between steps of a sharded handle");
  g->step_with_barrier = with_barrier; g->step_mode = 0;
  if (N == 0) { g->step_in_flight = true; return SB200_OK; }
  const uint4* oldr = (const uint4*)g->regs[g->cur].p;
  uint4* newr = (uint4*)g->regs[g->cur ^ 1].p;
  const uint32_t* bmp = g->bm[g->bcur].p;
  uint32_t* bmc = g->bm[g->bcur ^ 1].p;
  const double dense_frac = g->dense_frac, push_div = g->push_div;
  const int force_mode = g->force_mode;
  int mode;
  const double E = (double)std::max<uint64_t>(g->E_kept, 1);
  if (g->world == 1) {
    // the source-major CSR is built lazily: when a reused handle (or a pinned push policy) first meets a frontier
    // of < N/64 nodes.  A handle that computes one centrality and is dropped never pays for it.
    if (!g->has_fwd && ((g->reuse > 0 && g->t > 0 && (double)g->n_changed_prev * 64.0 <= (double)N) || force_mode == 2)) {
      SB_TRY(build_fwd_csr(g));
      SB_CUDA(cudaMemsetAsync(g->counters.p + 4, 0, sizeof(unsigned long long), s));
      SB_LAUNCH(k_frontier_out_edges, div_up(words, 256), 256, 0, s, bmp, words, g->fwd_ptr.p, g->counters.p + 4);
      SB_CHECK_LAUNCH();
      unsigned long long fe0 = 0;
      SB_CUDA(cudaMemcpyAsync(&fe0, g->counters.p + 4, sizeof(fe0), cudaMemcpyDeviceToHost, s));
      SB_CUDA(cudaStreamSynchronize(s));
      g->frontier_edges_prev = fe0;
    }
    if (g->has_fwd) {
      const double fe = (double)g->frontier_edges_prev;
      if (fe >= dense_frac * E) mode = 0;
      else if (fe * push_div <= E) mode = 2;
      else mode = 1;
    } else {
      mode = ((double)g->n_changed_prev >= 0.75 * (double)N) ? 0 : 1;
    }
  } else {
    // sharded handles: the same lazy rule for the source-major CSR (of the owned rows); every rank sees the same
    // global changed count, so all ranks switch together
    // Thresholds: below 0.75 N changed nodes a frontier-filtered pull reads fewer source registers than a dense one (the
    // rule of a single rank without forward CSR); below N / 16 a push over the changed rows' out-edges does less work than a
    // frontier pull, which still scans every local edge.
    const bool tiny = (double)g->n_changed_prev * 16.0 <= (double)N;
    if (!g->has_fwd && ((g->reuse > 0 && g->t > 0 && tiny) || force_mode == 2)) SB_TRY(build_fwd_csr(g));
    if (g->has_fwd && tiny) mode = 2;
    else mode = ((double)g->n_changed_prev >= 0.75 * (double)N) ? 0 : 1;
  }
  if (force_mode >= 0 && (force_mode < 2 || g->has_fwd)) mode = force_mode;
  g->step_mode = mode;
  SB_CUDA(cudaEventRecord(g->ev0, s));
  // peers write their changed bits straight into this rank's bitmap, so with the fused exchange it is cleared
  // at the END of the previous step (before the inter-step barrier), never at the start of this one
  if (!g->p2p) SB_CUDA(cudaMemsetAsync(bmc, 0, (words + 1) * 4, s));
  SB_CUDA(cudaMemsetAsync(g->counters.p, 0, 8 * sizeof(unsigned long long), s));
  // Iteration 0 pulls from the seeds.  Invariant: at t = 0 every row of regs[cur] is the one-hot row of its seed --
  // hb_reset writes both from one hash (create and bind_state end in hb_reset), and no call writes registers between
  // a reset and the first step.  bm_prev is all ones at t = 0, so a forced frontier pull is the same pull; a forced
  // push keeps its path.
  const bool from_seed = g->t == 0 && mode != 2;
  if (g->l2_window_bytes && mode != 2) {
    const void* wbase; uint64_t wbytes;
    l2_window_of(g, oldr, from_seed, &wbase, &wbytes);
    SB_TRY(set_l2_window(s, wbase, wbytes));
  }
  if (from_seed) SB_TRY((launch_pull<false, true>(g, oldr, newr, bmp, bmc)));
  else if (mode == 0) SB_TRY((launch_pull<false, false>(g, oldr, newr, bmp, bmc)));
  else if (mode == 1) SB_TRY((launch_pull<true, false>(g, oldr, newr, bmp, bmc)));
  else SB_TRY(run_push(g, oldr, newr, bmp, bmc));
  if (g->p2p && g->n_peers > 0) {
    const PeerOut po = make_peer_out(g, true);
    SB_LAUNCH(k_publish_bitmap, div_up(words, 256), 256, 0, s, bmc, words, po);
    SB_CHECK_LAUNCH();
  }
  PROF_BEGIN(g, sb200_graph::F_FINALIZE);
  if (!g->sm_count) SB_CUDA(cudaDeviceGetAttribute(&g->sm_count, cudaDevAttrMultiProcessorCount, g->device));
  const unsigned fin_grid = (unsigned)std::min<uint64_t>(div_up(div_up(N, (uint64_t)std::max(g->world, 1)), 256) + 1, (uint64_t)g->sm_count * 8);
  SB_LAUNCH(k_finalize, fin_grid, 256, 0, s, (uint64_t)0, N, newr, bmp, bmc, g->size_cache.p,
            g->kahan_sum.p, g->kahan_err.p, g->has_fwd ? g->fwd_ptr.p : (const uint32_t*)nullptr, (double)(g->t + 1),
            g->counters.p, (uint32_t)g->world, (uint32_t)g->rank);
  SB_CHECK_LAUNCH();
  PROF_END(g, sb200_graph::F_FINALIZE, 0.25 * (double)N);  // 2 bitmap bits/row; + 112 B per changed row below
  if (g->p2p) SB_CUDA(cudaMemsetAsync((void*)bmp, 0, (words + 1) * 4, s));  // next step's `cur` bitmap
  if (with_barrier) {
    if (!g->sync_page.p || g->n_peers != g->world - 1) SB_FAIL(SB200_ESTATE, "device barrier needs the sync pages of all %d peers", g->world - 1);
    g->sync_epoch++;
    SB_LAUNCH(k_barrier_count, 1, 32, 0, s, make_sync_view(g), (unsigned long long)g->sync_epoch, (const unsigned long long*)g->counters.p,
              g->counters.p + 5, 20000000000ull);
    SB_CHECK_LAUNCH();
  }
  SB_CUDA(cudaMemcpyAsync(g->h_counters, g->counters.p, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  SB_CUDA(cudaEventRecord(g->ev1, s));
  g->step_in_flight = true;
  return SB200_OK;
}

int hb_step_finish(sb200_graph* g, sb200_iter_stats* st) {
  NvtxRange nvtx("sb200 hyperball iteration (wait)");
  cudaStream_t s = g->stream;
  if (!g->step_in_flight) SB_FAIL(SB200_ESTATE, "no step in flight");
  g->step_in_flight = false;
  if (g->N == 0) { g->has_changes = false; if (st) memset(st, 0, sizeof(*st)); return SB200_OK; }
  SB_CUDA(cudaStreamSynchronize(s));
  float ms = 0; cudaEventElapsedTime(&ms, g->ev0, g->ev1);
  if (g->profiling) {
    g->prof_step_bytes[sb200_graph::F_FINALIZE] += 112.0 * (double)g->h_counters[0];
    for (int f = 0; f < sb200_graph::F_COUNT; f++) if (g->prof_used[f]) {
      float kms = 0; cudaEventElapsedTime(&kms, g->prof_ev[f][0], g->prof_ev[f][1]);
      g->prof_launches[f]++; g->prof_ms[f] += kms; g->prof_bytes[f] += g->prof_step_bytes[f];
      g->prof_used[f] = false;
    }
    if (g->side_prof_used) {
      const int f = g->side_prof_family;
      float kms = 0; cudaEventElapsedTime(&kms, g->side_prof[0], g->side_prof[1]);
      g->prof_launches[f]++; g->prof_ms[f] += kms; g->prof_bytes[f] += g->prof_step_bytes[f];
      g->side_prof_used = false;
    }
  }
  if (st) {
    st->t = g->t; st->mode = (uint32_t)g->step_mode; st->n_changed = g->h_counters[0];
    st->edges_active = g->frontier_edges_prev; st->ms = ms;
  }
  g->cur ^= 1; g->bcur ^= 1; g->t += 1;
  if (g->world == 1) {
    g->n_changed_prev = g->h_counters[0];
    g->frontier_edges_prev = g->h_counters[1];
    g->has_changes = g->h_counters[0] != 0;
  } else if (g->step_with_barrier) {
    if (g->h_counters[6]) SB_FAIL(SB200_ESTATE, "inter-rank barrier timed out in iteration %u: %llu rank(s) did not arrive", g->t - 1, (unsigned long long)g->h_counters[6]);
    g->n_changed_prev = g->h_counters[5];   // the global count, summed on the device
    g->has_changes = g->h_counters[5] != 0;
  } else {
    g->n_changed_prev = g->h_counters[0];
    g->exchange_pending = true;
  }
  return SB200_OK;
}

int hb_step(sb200_graph* g, sb200_iter_stats* st) {
  SB_TRY(hb_step_launch(g, false));
  return hb_step_finish(g, st);
}

int hb_result(sb200_graph* g, uint64_t* id_lo, uint64_t* id_hi, double* cent, uint64_t cap, uint64_t* len) {
  NvtxRange nvtx("sb200 hyperball result");
  cudaStream_t s = g->stream;
  const uint64_t N = g->N;
  if (N == 0) { *len = 0; return SB200_OK; }
  PoolScope scope(getenv("SB200_NO_POOL") ? nullptr : s);  // temporaries from the stream-ordered pool, freed on `s`
  const auto tp0 = std::chrono::steady_clock::now();
  DevBuf<uint32_t> flag, pos; DevBuf<double> val;
  SB_TRY(flag.alloc(N + 1)); SB_TRY(pos.alloc(N + 1)); SB_TRY(val.alloc(N));
  SB_CUDA(cudaMemsetAsync(flag.p + N, 0, 4, s));
  const double norm = (double)(N - 1);
  SB_LAUNCH(k_result_flags, div_up(N, 256), 256, 0, s, g->inv.p, g->kahan_sum.p, N, (uint64_t)0, N, norm, flag.p, val.p,
            (uint32_t)g->world, (uint32_t)g->rank);
  SB_CHECK_LAUNCH();
  size_t need = 0;
  SB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, need, flag.p, pos.p, (int64_t)(N + 1), s));
  if (g->cub_tmp.n < need) SB_TRY(g->cub_tmp.alloc(need + 256));
  SB_CUDA(cub::DeviceScan::ExclusiveSum(g->cub_tmp.p, need, flag.p, pos.p, (int64_t)(N + 1), s));
  g_launches.fetch_add(2, std::memory_order_relaxed);
  uint32_t total = 0;
  SB_CUDA(cudaMemcpyAsync(&total, pos.p + N, 4, cudaMemcpyDeviceToHost, s));
  SB_CUDA(cudaStreamSynchronize(s));
  const bool timing = getenv("SB200_RESULT_TIMING") != nullptr;
  const auto tp1 = std::chrono::steady_clock::now();
  if (timing) fprintf(stderr, "[sb200 result] flags+scan %.2f ms\n", std::chrono::duration<double, std::milli>(tp1 - tp0).count());
  *len = total;
  if (!cent) return SB200_OK;
  const uint64_t k = std::min<uint64_t>(total, cap);
  if (k == 0) return SB200_OK;
  DevBuf<uint64_t> olo, ohi; DevBuf<double> oc;
  SB_TRY(olo.alloc(k)); SB_TRY(ohi.alloc(k)); SB_TRY(oc.alloc(k));
  SB_LAUNCH(k_result_scatter, div_up(N, 256), 256, 0, s, flag.p, pos.p, val.p, g->id_lo.p, g->id_hi.p, N, k, olo.p, ohi.p, oc.p);
  SB_CHECK_LAUNCH();
  SB_CUDA(cudaMemcpyAsync(id_lo, olo.p, k * 8, cudaMemcpyDefault, s));
  SB_CUDA(cudaMemcpyAsync(id_hi, ohi.p, k * 8, cudaMemcpyDefault, s));
  SB_CUDA(cudaMemcpyAsync(cent, oc.p, k * 8, cudaMemcpyDefault, s));
  SB_CUDA(cudaStreamSynchronize(s));
  if (timing) fprintf(stderr, "[sb200 result] scatter+d2h of %llu rows %.2f ms\n", (unsigned long long)k,
                      std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tp1).count());
  return SB200_OK;
}

// ---- rank assignment (store_harmonic's second pass, crates/core/src/webgraph/centrality/mod.rs:88-108) -----------
// key = ~order-preserving bits of the centrality (ascending key == descending f64 total order); the stable radix sort
// keeps the input order among equal keys, so feeding the nodes in ascending (descending) id order yields the
// (centrality desc, id asc) order of the rank store, or top_nodes' (centrality, id) descending order (mod.rs:17-37)
__global__ void k_rank_keys(const uint32_t* __restrict__ flag, const uint32_t* __restrict__ pos, const double* __restrict__ val,
                            uint64_t N, uint32_t total, int ties_desc, uint64_t* keys, uint32_t* ranks) {
  const uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (r >= N || !flag[r]) return;
  const uint32_t p = ties_desc ? total - 1u - pos[r] : pos[r];
  const uint64_t b = (uint64_t)__double_as_longlong(val[r]);
  keys[p] = ~((b >> 63) ? ~b : (b | 0x8000000000000000ull));
  ranks[p] = (uint32_t)r;
}
__global__ void k_rank_gather(const uint32_t* __restrict__ order, const double* __restrict__ val, const uint64_t* __restrict__ id_lo,
                              const uint64_t* __restrict__ id_hi, uint64_t k, uint64_t* out_lo, uint64_t* out_hi, double* out_c) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= k) return;
  const uint32_t r = order[i];
  out_lo[i] = id_lo[r]; out_hi[i] = id_hi[r]; out_c[i] = val[r];
}

int hb_ranked(sb200_graph* g, int ties_desc, uint64_t* id_lo, uint64_t* id_hi, double* cent, uint64_t cap, uint64_t* len) {
  cudaStream_t s = g->stream;
  const uint64_t N = g->N;
  if (g->world != 1) SB_FAIL(SB200_ESTATE, "ranking needs every node: gather the sharded results first");
  if (N == 0) { *len = 0; return SB200_OK; }
  PoolScope scope(getenv("SB200_NO_POOL") ? nullptr : s);
  DevBuf<uint32_t> flag, pos; DevBuf<double> val;
  SB_TRY(flag.alloc(N + 1)); SB_TRY(pos.alloc(N + 1)); SB_TRY(val.alloc(N));
  SB_CUDA(cudaMemsetAsync(flag.p + N, 0, 4, s));
  SB_LAUNCH(k_result_flags, div_up(N, 256), 256, 0, s, g->inv.p, g->kahan_sum.p, N, (uint64_t)0, N, (double)(N - 1), flag.p,
            val.p, 1u, 0u);
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
  if (!cent || k == 0) return SB200_OK;
  DevBuf<uint64_t> ka, kb; DevBuf<uint32_t> va, vb;
  SB_TRY(ka.alloc(total)); SB_TRY(kb.alloc(total)); SB_TRY(va.alloc(total)); SB_TRY(vb.alloc(total));
  SB_LAUNCH(k_rank_keys, div_up(N, 256), 256, 0, s, flag.p, pos.p, val.p, N, total, ties_desc, ka.p, va.p);
  SB_CHECK_LAUNCH();
  cub::DoubleBuffer<uint64_t> dk(ka.p, kb.p);
  cub::DoubleBuffer<uint32_t> dv(va.p, vb.p);
  need = 0;
  SB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, need, dk, dv, (int64_t)total, 0, 64, s));
  if (g->cub_tmp.n < need) SB_TRY(g->cub_tmp.alloc(need + 256));
  SB_CUDA(cub::DeviceRadixSort::SortPairs(g->cub_tmp.p, need, dk, dv, (int64_t)total, 0, 64, s));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  DevBuf<uint64_t> olo, ohi; DevBuf<double> oc;
  SB_TRY(olo.alloc(k)); SB_TRY(ohi.alloc(k)); SB_TRY(oc.alloc(k));
  SB_LAUNCH(k_rank_gather, div_up(k, 256), 256, 0, s, dv.Current(), val.p, g->id_lo.p, g->id_hi.p, k, olo.p, ohi.p, oc.p);
  SB_CHECK_LAUNCH();
  SB_CUDA(cudaMemcpyAsync(id_lo, olo.p, k * 8, cudaMemcpyDefault, s));
  SB_CUDA(cudaMemcpyAsync(id_hi, ohi.p, k * 8, cudaMemcpyDefault, s));
  SB_CUDA(cudaMemcpyAsync(cent, oc.p, k * 8, cudaMemcpyDefault, s));
  SB_CUDA(cudaStreamSynchronize(s));
  return SB200_OK;
}

int hb_registers(sb200_graph* g, uint64_t first, uint64_t count, uint8_t* out) {
  if (first + count > g->N) SB_FAIL(SB200_EINVAL, "register range [%llu,+%llu) outside %llu nodes", (unsigned long long)first, (unsigned long long)count, (unsigned long long)g->N);
  if (!count) return SB200_OK;
  DevBuf<uint4> tmp; SB_TRY(tmp.alloc(count * 4));
  SB_LAUNCH(k_gather_regs, div_up(count * 4, 256), 256, 0, g->stream, g->inv.p, (const uint4*)g->regs[g->cur].p, first, count, tmp.p);
  SB_CHECK_LAUNCH();
  SB_CUDA(cudaMemcpyAsync(out, tmp.p, count * 64, cudaMemcpyDefault, g->stream));
  SB_CUDA(cudaStreamSynchronize(g->stream));
  return SB200_OK;
}
int hb_kahan(sb200_graph* g, uint64_t first, uint64_t count, double* sum, double* err) {
  if (first + count > g->N) SB_FAIL(SB200_EINVAL, "range outside the node set");
  if (!count) return SB200_OK;
  DevBuf<double> a, b; SB_TRY(a.alloc(count)); SB_TRY(b.alloc(count));
  SB_LAUNCH(k_gather_f64x2, div_up(count, 256), 256, 0, g->stream, g->inv.p, g->kahan_sum.p, g->kahan_err.p, first, count, a.p, b.p);
  SB_CHECK_LAUNCH();
  SB_CUDA(cudaMemcpyAsync(sum, a.p, count * 8, cudaMemcpyDefault, g->stream));
  SB_CUDA(cudaMemcpyAsync(err, b.p, count * 8, cudaMemcpyDefault, g->stream));
  SB_CUDA(cudaStreamSynchronize(g->stream));
  return SB200_OK;
}

}  // namespace sb200
