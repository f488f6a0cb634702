// graph_stage.cu -- staging of the webgraph edge stream into HBM.
//
// Replaces, on the device, what the reference does on one CPU thread every time it scans the
// graph: `Webgraph::host_nodes()` (FxHashSet of all endpoints, crates/core/src/webgraph/mod.rs:157,
// store.rs:338-357), `host_edges()` + `unique_by((from,to))` (store.rs:297-315) and the
// `BTreeMap<NodeID,_>` keyed lookups of harmonic.rs:134-135.  Here it happens once:
//   1. u128 node ids -> open-addressing hash set in HBM (128-bit CAS), compacted and sorted
//      ascending => dense rank (the BTreeMap order of the reference's output);
//   2. every edge mapped to (to_rank<<32 | from_rank), stable radix sort, first-of-run keeps the
//      FIRST occurrence's rel_flags (unique_by semantics), skipped / self-loop edges dropped;
//   3. nodes relabelled by in-degree (descending) so that rows of equal length are adjacent:
//      the degree classes of the pull kernels become contiguous row ranges; the rows of the
//      sorted keys move as blocks to their new place (k_row_permute).  The source-major CSR of the
//      small-frontier (push) branch is built lazily from the resident one (build_fwd_csr).
// Radix sorts / scans / selects are CUB device primitives (staging, not the hot loop).
#include "graph.cuh"

#ifndef SB200_EMU
#include <cub/cub.cuh>
#endif
#include <algorithm>
#include <ctime>
#include <cstdlib>

namespace sb200 {

typedef unsigned __int128 u128;

__device__ __forceinline__ u128 cas128(u128* addr, u128 cmp, u128 val) {
#ifndef SB200_EMU
  u128 old;
  asm volatile("atom.global.cas.b128 %0, [%1], %2, %3;" : "=q"(old) : "l"(addr), "q"(cmp), "q"(val) : "memory");
  return old;
#else
  const u128 old = *addr;   // tests/emu runs one thread at a time
  if (old == cmp) *addr = val;
  return old;
#endif
}
__device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ uint64_t hash128(uint64_t lo, uint64_t hi) {
  return mix64(lo ^ (hi * 0x9E3779B97F4A7C15ull) ^ (hi >> 29));
}
#define EMPTY64 0xFFFFFFFFFFFFFFFFull

// inserts one endpoint and returns the table slot that holds it (0xFFFFFFFF for the all-ones id / on overflow)
// flags: [0] overflow, [1] the all-ones id is present (it doubles as the empty sentinel)
__device__ __forceinline__ uint32_t insert_slot(ulonglong2* table, uint64_t mask, uint64_t lo, uint64_t hi,
                                                unsigned long long* count, unsigned long long max_count, int* flags) {
  if (lo == EMPTY64 && hi == EMPTY64) { flags[1] = 1; return 0xFFFFFFFFu; }
  const u128 key = ((u128)hi << 64) | lo;
  uint64_t slot = hash128(lo, hi) & mask;
  for (uint64_t probe = 0;; probe++) {
    const ulonglong2 cur = table[slot];
    if (cur.x == lo && cur.y == hi) return (uint32_t)slot;
    if (cur.x == EMPTY64 || cur.y == EMPTY64) {
      // empty, being written, or a key with an all-ones half: the CAS result is the truth
      const u128 old = cas128((u128*)&table[slot], ~(u128)0, key);
      if (old == ~(u128)0) {
        const unsigned long long c = atomicAdd(count, 1ull);
        if (c + 1 > max_count) flags[0] = 1;
        return (uint32_t)slot;
      }
      if (old == key) return (uint32_t)slot;
    }
    slot = (slot + 1) & mask;
    if (probe > mask) { flags[0] = 1; return 0xFFFFFFFFu; }
  }
}
__global__ void k_insert_edges(const uint64_t* __restrict__ flo, const uint64_t* __restrict__ fhi,
                               const uint64_t* __restrict__ tlo, const uint64_t* __restrict__ thi,
                               const uint64_t* __restrict__ rel, uint64_t n, uint64_t skip_mask, ulonglong2* table,
                               uint64_t mask, unsigned long long* count, unsigned long long max_count, int* flags,
                               uint32_t* slot_from, uint32_t* slot_to, uint8_t* skip) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    if (*(volatile int*)flags) return;  // table overflow: the host grows it and replays the stream
    slot_from[i] = insert_slot(table, mask, flo[i], fhi[i], count, max_count, flags);
    slot_to[i] = insert_slot(table, mask, tlo[i], thi[i], count, max_count, flags);
    skip[i] = (rel[i] & skip_mask) != 0;
  }
}
__global__ void k_map_slots(const uint32_t* __restrict__ slot_from, const uint32_t* __restrict__ slot_to, uint64_t n,
                            const uint32_t* __restrict__ slot_val, uint32_t max_rank, uint64_t* keys) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t sf = slot_from[i], st = slot_to[i];
  const uint32_t rf = sf == 0xFFFFFFFFu ? max_rank : slot_val[sf];
  const uint32_t rt = st == 0xFFFFFFFFu ? max_rank : slot_val[st];
  keys[i] = ((uint64_t)rt << 32) | rf;
}

__global__ void k_compact_keys(const ulonglong2* __restrict__ table, uint64_t cap, uint64_t* out_lo,
                               uint64_t* out_hi, unsigned long long* counter) {
  for (uint64_t base = blockIdx.x * (uint64_t)blockDim.x; base < cap; base += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t i = base + threadIdx.x;
    ulonglong2 cur = make_ulonglong2(EMPTY64, EMPTY64);
    if (i < cap) cur = table[i];
    bool occ = !(cur.x == EMPTY64 && cur.y == EMPTY64);
    unsigned m = __ballot_sync(0xffffffffu, occ);
    int lane = threadIdx.x & 31;
    unsigned long long wbase = 0;
    if (lane == 0 && m) wbase = atomicAdd(counter, (unsigned long long)__popc(m));
    wbase = __shfl_sync(0xffffffffu, wbase, 0);
    if (occ) {
      uint64_t pos = wbase + __popc(m & ((1u << lane) - 1));
      out_lo[pos] = cur.x; out_hi[pos] = cur.y;
    }
  }
}

__global__ void k_assign_ranks(const uint64_t* __restrict__ lo, const uint64_t* __restrict__ hi, uint64_t n,
                               const ulonglong2* __restrict__ table, uint32_t* slot_val, uint64_t mask) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t l = lo[i], h = hi[i];
  uint64_t slot = hash128(l, h) & mask;
  for (;;) {
    ulonglong2 cur = table[slot];
    if (cur.x == l && cur.y == h) { slot_val[slot] = (uint32_t)i; return; }
    slot = (slot + 1) & mask;
  }
}

__global__ void k_mark_keep(const uint64_t* __restrict__ keys, const uint8_t* __restrict__ skip, uint64_t n,
                            uint8_t* keep, uint32_t* self_bm) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t k = keys[i];
  bool first = (i == 0) || (keys[i - 1] != k);
  const bool self = (uint32_t)k == (uint32_t)(k >> 32);
  keep[i] = first && !skip[i] && !self;
  if (first && !skip[i] && self) atomicOr(self_bm + ((uint32_t)k >> 5), 1u << ((uint32_t)k & 31u));   // kept self-link: remembered, not stored
}

__global__ void k_degree_hi(const uint64_t* __restrict__ keys, uint64_t n, uint32_t* deg) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) atomicAdd(&deg[keys[i] >> 32], 1u);
}
__global__ void k_iota(uint32_t* a, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) a[i] = (uint32_t)i;
}
__global__ void k_invert(const uint32_t* __restrict__ perm, uint64_t n, uint32_t* inv) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) inv[perm[i]] = (uint32_t)i;
}
// Relabelling permutes whole CSR rows: the rank-space keys are already grouped by destination, so row `to` (edges
// [rank_ptr[to], rank_ptr[to+1])) moves as a block to row_ptr[inv[to]] and only the source ids are translated.
// One pass instead of a second 64-bit radix sort of all edges.  Sources inside a row stay in rank order instead of
// internal-id order; the pull kernels take a max over them, so the order is immaterial.
__global__ void k_row_permute(const uint64_t* __restrict__ keys, uint64_t n, const uint32_t* __restrict__ rank_ptr,
                              const uint32_t* __restrict__ inv, const uint32_t* __restrict__ row_ptr, uint32_t* col) {
  const uint64_t e = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (e >= n) return;
  const uint64_t k = keys[e];
  const uint32_t to = (uint32_t)(k >> 32);
  col[(uint64_t)row_ptr[inv[to]] + (e - rank_ptr[to])] = inv[(uint32_t)k];
}
__global__ void k_lo32(const uint64_t* __restrict__ in, uint64_t n, uint32_t* out) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = (uint32_t)in[i];
}
// deg is sorted descending: count rows with deg > thresholds[j] by boundary detection
__global__ void k_class_bounds(const uint32_t* __restrict__ deg, uint64_t n, uint32_t t0, uint32_t t1,
                               uint32_t t2, unsigned long long* out) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t d = deg[i];
  uint32_t nx = (i + 1 < n) ? deg[i + 1] : 0u;
  if (d > t0 && !(nx > t0)) out[0] = i + 1;
  if (d > t1 && !(nx > t1)) out[1] = i + 1;
  if (d > t2 && !(nx > t2)) out[2] = i + 1;
}
__global__ void k_owned_edges(const uint32_t* __restrict__ row_ptr, uint64_t n, uint32_t world, uint32_t rank,
                              unsigned long long* out) {
  const uint64_t v = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  unsigned long long d = 0;
  if (v < n && ((v >> 5) % world) == rank) d = row_ptr[v + 1] - row_ptr[v];
  for (int o = 16; o; o >>= 1) d += __shfl_down_sync(0xffffffffu, d, o);
  if ((threadIdx.x & 31) == 0 && d) atomicAdd(out, d);
}
// Subscriber masks (sharded handles): bit r of sub[u] is set iff some row owned by rank r has an in-edge from u, i.e.
// rank r gathers u's counter.  The test before the atomic keeps the ~E updates of a power-law graph from piling up on
// the hubs' words: once a bit is set, later edges only read it.
__device__ __forceinline__ void sub_mark(uint32_t* sub, uint32_t u, uint32_t bit) {
  if ((__ldg(sub + u) & bit) == 0u) atomicOr(sub + u, bit);
}
__global__ void k_sub_items(uint64_t n_items, const uint32_t* __restrict__ item_row, const uint32_t* __restrict__ item_start,
                            uint32_t warp_row_begin, const uint32_t* __restrict__ row_ptr, const uint32_t* __restrict__ col, int chunk,
                            uint32_t world, uint32_t* sub) {
  const uint64_t item = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  if (item >= n_items) return;
  const uint32_t lane = threadIdx.x & 31, row = item_row[item];
  const uint32_t bit = 1u << ((row >> 5) % world);
  const uint32_t c = (uint32_t)item - item_start[row - warp_row_begin];
  const uint32_t e0 = row_ptr[row] + c * (uint32_t)chunk, e1 = min(e0 + (uint32_t)chunk, row_ptr[row + 1]);
  for (uint32_t e = e0 + lane; e < e1; e += 32) sub_mark(sub, col[e], bit);
}
__global__ void k_sub_rows(uint64_t row_begin, uint64_t row_end, const uint32_t* __restrict__ row_ptr, const uint32_t* __restrict__ col,
                           uint32_t world, uint32_t* sub) {
  const uint64_t row = row_begin + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (row >= row_end) return;
  const uint32_t bit = 1u << ((uint32_t)(row >> 5) % world);
  for (uint32_t e = row_ptr[row]; e < row_ptr[row + 1]; e++) sub_mark(sub, col[e], bit);
}
// remote subscribers of the rows this rank owns (the number of 64-B rows one dense iteration sends over NVLink)
__global__ void k_sub_count(const uint32_t* __restrict__ sub, uint64_t n, uint32_t world, uint32_t rank, unsigned long long* out) {
  const uint64_t v = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  unsigned long long d = 0;
  if (v < n && ((v >> 5) % world) == rank) d = __popc(sub[v] & ~(1u << rank));
  for (int o = 16; o; o >>= 1) d += __shfl_down_sync(0xffffffffu, d, o);
  if ((threadIdx.x & 31) == 0 && d) atomicAdd(out, d);
}
__global__ void k_row_chunks(const uint32_t* __restrict__ row_ptr, uint64_t row0, uint64_t nrows, int chunk,
                             uint32_t* nchunks) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= nrows) return;
  uint32_t d = row_ptr[row0 + i + 1] - row_ptr[row0 + i];
  nchunks[i] = (d + chunk - 1) / chunk;
}
// sharded handles: the work items of the rows this rank owns, ascending (so k_pull_warp launches no warp that would exit)
__global__ void k_item_owned_flag(uint64_t n_items, const uint32_t* __restrict__ item_row, uint32_t world, uint32_t rank, uint32_t* flag) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i > n_items) return;
  flag[i] = (i < n_items && ((item_row[i] >> 5) % world) == rank) ? 1u : 0u;
}
__global__ void k_item_owned_scatter(uint64_t n_items, const uint32_t* __restrict__ flag, const uint32_t* __restrict__ pos, uint32_t* list) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n_items && flag[i]) list[pos[i]] = (uint32_t)i;
}
__global__ void k_fill_items(const uint32_t* __restrict__ item_start, uint64_t nrows, uint64_t n_items,
                             uint32_t row0, uint32_t* item_row) {
  uint64_t it = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (it >= n_items) return;
  uint64_t lo = 0, hi = nrows;  // last row r with item_start[r] <= it
  while (lo + 1 < hi) { uint64_t mid = (lo + hi) / 2; if (item_start[mid] <= it) lo = mid; else hi = mid; }
  item_row[it] = row0 + (uint32_t)lo;
}

bool is_device_ptr(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}
int copy_in(void* dst, const void* src, size_t bytes, cudaStream_t s) {
  if (bytes == 0) return SB200_OK;
  SB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, s));
  return SB200_OK;
}

// (src<<32 | dst) key of every edge of the resident destination-major CSR: short rows one thread per row, long
// rows one warp per work item
__global__ void k_fwd_keys_rows(uint64_t row_begin, uint64_t row_end, const uint32_t* __restrict__ row_ptr,
                                const uint32_t* __restrict__ col, uint64_t* keys) {
  const uint64_t row = row_begin + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (row >= row_end) return;
  for (uint32_t e = row_ptr[row]; e < row_ptr[row + 1]; e++) keys[e] = ((uint64_t)col[e] << 32) | (uint32_t)row;
}
__global__ void k_fwd_keys_items(uint64_t n_items, const uint32_t* __restrict__ item_row, const uint32_t* __restrict__ item_start,
                                 uint32_t warp_row_begin, const uint32_t* __restrict__ row_ptr, const uint32_t* __restrict__ col,
                                 int chunk, uint64_t* keys) {
  const uint64_t item = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  if (item >= n_items) return;
  const uint32_t lane = threadIdx.x & 31, row = item_row[item];
  const uint32_t c = (uint32_t)item - item_start[row - warp_row_begin];
  const uint32_t e0 = row_ptr[row] + c * (uint32_t)chunk, e1 = min(e0 + (uint32_t)chunk, row_ptr[row + 1]);
  for (uint32_t e = e0 + lane; e < e1; e += 32) keys[e] = ((uint64_t)col[e] << 32) | row;
}
// sharded handles: the same keys for the OWNED destination rows only (interleaved 32-row blocks), written densely
// through own_ptr = exclusive scan of the owned in-degrees
__global__ void k_owned_deg(const uint32_t* __restrict__ row_ptr, uint64_t n, uint32_t world, uint32_t rank, uint32_t* deg) {
  const uint64_t v = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (v > n) return;
  deg[v] = (v < n && ((v >> 5) % world) == rank) ? row_ptr[v + 1] - row_ptr[v] : 0u;
}
__global__ void k_fwd_keys_rows_own(uint64_t row_begin, uint64_t row_end, const uint32_t* __restrict__ row_ptr,
                                    const uint32_t* __restrict__ own_ptr, const uint32_t* __restrict__ col, uint32_t world,
                                    uint32_t rank, uint64_t* keys) {
  const uint64_t row = row_begin + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (row >= row_end || ((row >> 5) % world) != rank) return;
  const uint32_t e0 = row_ptr[row], e1 = row_ptr[row + 1], o0 = own_ptr[row];
  for (uint32_t e = e0; e < e1; e++) keys[o0 + (e - e0)] = ((uint64_t)col[e] << 32) | (uint32_t)row;
}
__global__ void k_fwd_keys_items_own(uint64_t n_items, const uint32_t* __restrict__ item_row, const uint32_t* __restrict__ item_start,
                                     uint32_t warp_row_begin, const uint32_t* __restrict__ row_ptr,
                                     const uint32_t* __restrict__ own_ptr, const uint32_t* __restrict__ col, int chunk,
                                     uint32_t world, uint32_t rank, uint64_t* keys) {
  const uint64_t item = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  if (item >= n_items) return;
  const uint32_t lane = threadIdx.x & 31, row = item_row[item];
  if (((row >> 5) % world) != rank) return;
  const uint32_t c = (uint32_t)item - item_start[row - warp_row_begin];
  const uint32_t r0 = row_ptr[row], e0 = r0 + c * (uint32_t)chunk, e1 = min(e0 + (uint32_t)chunk, row_ptr[row + 1]);
  const uint32_t o0 = own_ptr[row];
  for (uint32_t e = e0 + lane; e < e1; e += 32) keys[o0 + (e - r0)] = ((uint64_t)col[e] << 32) | row;
}
// CSR offsets from keys sorted by their high word: ptr[r] = first index whose row >= r (no atomics)
__global__ void k_offsets_from_sorted(const uint64_t* __restrict__ keys, uint64_t n, uint64_t n_rows, uint32_t* ptr) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i > n) return;
  const uint64_t r = (i < n) ? (keys[i] >> 32) : n_rows;
  const uint64_t rp = (i == 0) ? 0 : (keys[i - 1] >> 32) + 1;
  for (uint64_t x = rp; x <= r && x <= n_rows; x++) ptr[x] = (uint32_t)i;
}

template <class K, class V>
static int sort_pairs(DevBuf<uint8_t>& tmp, K*& k, K*& k_alt, V*& v, V*& v_alt, uint64_t n, int b0, int b1,
                      bool descending, cudaStream_t s) {
  cub::DoubleBuffer<K> dk(k, k_alt);
  cub::DoubleBuffer<V> dv(v, v_alt);
  size_t need = 0;
  if (descending) SB_CUDA(cub::DeviceRadixSort::SortPairsDescending(nullptr, need, dk, dv, (int64_t)n, b0, b1, s));
  else SB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, need, dk, dv, (int64_t)n, b0, b1, s));
  if (tmp.n < need) SB_TRY(tmp.alloc(need + (need >> 3) + 256));
  if (descending) SB_CUDA(cub::DeviceRadixSort::SortPairsDescending(tmp.p, need, dk, dv, (int64_t)n, b0, b1, s));
  else SB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, need, dk, dv, (int64_t)n, b0, b1, s));
  g_launches.fetch_add(8, std::memory_order_relaxed);
  if (dk.Current() != k) std::swap(k, k_alt);
  if (dv.Current() != v) std::swap(v, v_alt);
  return SB200_OK;
}
template <class K>
static int sort_keys(DevBuf<uint8_t>& tmp, K*& k, K*& k_alt, uint64_t n, int b0, int b1, cudaStream_t s) {
  cub::DoubleBuffer<K> dk(k, k_alt);
  size_t need = 0;
  SB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, need, dk, (int64_t)n, b0, b1, s));
  if (tmp.n < need) SB_TRY(tmp.alloc(need + (need >> 3) + 256));
  SB_CUDA(cub::DeviceRadixSort::SortKeys(tmp.p, need, dk, (int64_t)n, b0, b1, s));
  g_launches.fetch_add(8, std::memory_order_relaxed);
  if (dk.Current() != k) std::swap(k, k_alt);
  return SB200_OK;
}
template <class T>
static int exclusive_scan_u32(DevBuf<uint8_t>& tmp, const T* in, uint32_t* out, uint64_t n, cudaStream_t s) {
  size_t need = 0;
  SB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, need, in, out, (int64_t)n, s));
  if (tmp.n < need) SB_TRY(tmp.alloc(need + 256));
  SB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, need, in, out, (int64_t)n, s));
  g_launches.fetch_add(2, std::memory_order_relaxed);
  return SB200_OK;
}

// optional per-phase wall timing of the staging pipeline (SB200_STAGE_TIMING=1 prints to stderr)
struct PhaseTimer {
  bool on; cudaStream_t s; double t0; const char* name = nullptr; const char* name_nvtx = nullptr;
#ifndef SB200_EMU
  ~PhaseTimer() { if (name_nvtx) nvtxRangePop(); }   // an early error return leaves no range open
#endif
  explicit PhaseTimer(cudaStream_t st) : s(st) { on = getenv("SB200_STAGE_TIMING") != nullptr; t0 = now(); }
  static double now() { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6; }
  void mark(const char* next) {
#ifndef SB200_EMU
    if (name_nvtx) nvtxRangePop();
    name_nvtx = next;
    if (next) nvtxRangePushA(next);
#endif
    if (!on) return;
    cudaStreamSynchronize(s);
    const double t = now();
    if (name) fprintf(stderr, "[sb200 stage] %-28s %9.2f ms\n", name, t - t0);
    name = next; t0 = t;
  }
};

static int bits_for(uint64_t n) { int b = 1; while (b < 32 && (1ull << b) < n) b++; return b; }

int stage_graph(sb200_graph* g, const uint64_t* from_lo, const uint64_t* from_hi, const uint64_t* to_lo,
                const uint64_t* to_hi, const uint64_t* rel, uint64_t n_edges, uint64_t skip_mask) {
  cudaStream_t s = g->stream;
  const int TPB = 256;
  g->E_in = n_edges;
  if (n_edges >= 0xFFFFFFF0ull) SB_FAIL(SB200_ERANGE, "n_edges %llu exceeds the 2^32-16 limit of u32 CSR offsets", (unsigned long long)n_edges);
  SB_CUDA(cudaEventRecord(g->ev0, s));
  PhaseTimer pt(s);
  pt.mark("0 copy-in");

  // ---- 0+1a. stream the SoA edge stream through HBM in chunks: while chunk c+1 crosses PCIe on the copy stream,
  //            the endpoints of chunk c are inserted into the node hash set and their table slots recorded.
  //            Only 9 B/edge (two u32 slots + the skip flag) stay resident instead of the 40 B/edge input.
  const uint64_t* src[5] = {from_lo, from_hi, to_lo, to_hi, rel};
  bool host_in[5];
  for (int a = 0; a < 5; a++) {
    if (n_edges && !src[a]) SB_FAIL(SB200_EINVAL, "edge array %d is NULL", a);
    host_in[a] = n_edges ? !is_device_ptr(src[a]) : false;
  }
  const uint64_t CHUNK = 1ull << 25;
  const uint64_t n_chunks = (n_edges + CHUNK - 1) / CHUNK;
  DevBuf<uint64_t> stg[2][5];
  for (int a = 0; a < 5; a++) if (host_in[a]) for (int bsel = 0; bsel < 2; bsel++) SB_TRY(stg[bsel][a].alloc(std::min<uint64_t>(CHUNK, n_edges)));
  struct Pipe {
    cudaStream_t cs = nullptr; cudaEvent_t copied[2] = {nullptr, nullptr}, consumed[2] = {nullptr, nullptr};
    ~Pipe() { for (int i = 0; i < 2; i++) { if (copied[i]) cudaEventDestroy(copied[i]); if (consumed[i]) cudaEventDestroy(consumed[i]); } if (cs) cudaStreamDestroy(cs); }
  } pipe;
  SB_CUDA(cudaStreamSynchronize(s));  // the staging buffers may be stream-ordered allocations of `s`; the copy stream uses them
  SB_CUDA(cudaStreamCreateWithFlags(&pipe.cs, cudaStreamNonBlocking));
  for (int i = 0; i < 2; i++) { SB_CUDA(cudaEventCreateWithFlags(&pipe.copied[i], cudaEventDisableTiming)); SB_CUDA(cudaEventCreateWithFlags(&pipe.consumed[i], cudaEventDisableTiming)); }

  DevBuf<unsigned long long> ctr; SB_TRY(ctr.alloc(8));
  DevBuf<int> flags; SB_TRY(flags.alloc(2));
  unsigned long long h_ctr[8]; int h_flags[2];
  DevBuf<uint8_t>& tmp = g->cub_tmp;
  DevBuf<uint32_t> slot_from, slot_to; SB_TRY(slot_from.alloc(n_edges)); SB_TRY(slot_to.alloc(n_edges));
  DevBuf<uint8_t> skip_a, skip_b; SB_TRY(skip_a.alloc(n_edges)); SB_TRY(skip_b.alloc(n_edges));

  // ---- 1. node dictionary ---------------------------------------------------------------------
  DevBuf<ulonglong2> table;
  uint64_t cap = 1ull << 12;
  while (cap < n_edges / 2) cap <<= 1;  // first guess: N <= E/4 keeps the load factor <= 1/2
  uint64_t n_keys = 0; bool has_max = false;
  for (;;) {
    SB_TRY(table.alloc(cap));
    SB_CUDA(cudaMemsetAsync(table.p, 0xFF, cap * sizeof(ulonglong2), s));
    SB_CUDA(cudaMemsetAsync(ctr.p, 0, 8 * sizeof(unsigned long long), s));
    SB_CUDA(cudaMemsetAsync(flags.p, 0, 2 * sizeof(int), s));
    for (uint64_t c = 0; c < n_chunks; c++) {
      const int bsel = (int)(c & 1);
      const uint64_t off = c * CHUNK, cnt = std::min<uint64_t>(CHUNK, n_edges - off);
      const uint64_t* ptr[5];
      bool any_host = false;
      for (int a = 0; a < 5; a++) {
        if (host_in[a]) {
          if (!any_host) SB_CUDA(cudaStreamWaitEvent(pipe.cs, pipe.consumed[bsel], 0));  // staging buffer free again
          any_host = true;
          SB_CUDA(cudaMemcpyAsync(stg[bsel][a].p, src[a] + off, cnt * 8, cudaMemcpyHostToDevice, pipe.cs));
          ptr[a] = stg[bsel][a].p;
        } else ptr[a] = src[a] + off;
      }
      if (any_host) { SB_CUDA(cudaEventRecord(pipe.copied[bsel], pipe.cs)); SB_CUDA(cudaStreamWaitEvent(s, pipe.copied[bsel], 0)); }
      const unsigned grid = (unsigned)std::min<uint64_t>(div_up(cnt, TPB), 148u * 32u);
      SB_LAUNCH(k_insert_edges, grid, TPB, 0, s, ptr[0], ptr[1], ptr[2], ptr[3], ptr[4], cnt, skip_mask, table.p, cap - 1, ctr.p,
                (unsigned long long)(cap / 2), flags.p, slot_from.p + off, slot_to.p + off, skip_a.p + off);
      SB_CHECK_LAUNCH();
      if (any_host) SB_CUDA(cudaEventRecord(pipe.consumed[bsel], s));
    }
    SB_CUDA(cudaMemcpyAsync(h_ctr, ctr.p, sizeof(h_ctr), cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaMemcpyAsync(h_flags, flags.p, sizeof(h_flags), cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaStreamSynchronize(s));
    SB_CUDA(cudaStreamSynchronize(pipe.cs));
    if (!h_flags[0]) { n_keys = h_ctr[0]; has_max = h_flags[1] != 0; break; }
    cap <<= 2;  // load factor exceeded 1/2: grow and redo (still linear overall)
    // slots are recorded as u32 and 0xFFFFFFFF is the sentinel (all-ones id / overflow), so the table must stay below
    // 2^32 slots: at most 2^31, i.e. <= 2^30 nodes at load factor 1/2 (n_edges < 2^32 keeps real inputs far below)
    if (cap > (1ull << 31)) SB_FAIL(SB200_ERANGE, "node hash set would exceed 2^31 slots (more than 2^30 distinct nodes)");
  }
  for (int a = 0; a < 5; a++) for (int bsel = 0; bsel < 2; bsel++) stg[bsel][a].release();
  pt.mark("1b compact+sort ids");
  const uint64_t N = n_keys + (has_max ? 1 : 0);
  g->N = N;
  if (N >= 0xFFFFFFFEull) SB_FAIL(SB200_ERANGE, "%llu nodes exceed the u32 index space", (unsigned long long)N);
  SB_TRY(g->id_lo.alloc(N)); SB_TRY(g->id_hi.alloc(N));
  SB_TRY(g->perm.alloc(N)); SB_TRY(g->inv.alloc(N));
  SB_TRY(g->row_ptr.alloc(N + 1));
  if (N == 0) {
    SB_CUDA(cudaMemsetAsync(g->row_ptr.p, 0, sizeof(uint32_t), s));
    g->E_kept = g->E_local = 0; g->n_pos = 0;
    SB_CUDA(cudaEventRecord(g->ev1, s)); SB_CUDA(cudaStreamSynchronize(s));
    return SB200_OK;
  }
  {
    // compact the occupied slots and sort ascending by (hi, lo): LSD = two stable 64-bit passes
    DevBuf<uint64_t> alt_lo, alt_hi; SB_TRY(alt_lo.alloc(N)); SB_TRY(alt_hi.alloc(N));
    SB_CUDA(cudaMemsetAsync(ctr.p, 0, sizeof(unsigned long long), s));
    unsigned grid = (unsigned)std::min<uint64_t>(div_up(cap, TPB), 148u * 32u);
    SB_LAUNCH(k_compact_keys, grid, TPB, 0, s, table.p, cap, g->id_lo.p, g->id_hi.p, ctr.p);
    SB_CHECK_LAUNCH();
    uint64_t *klo = g->id_lo.p, *klo_alt = alt_lo.p, *khi = g->id_hi.p, *khi_alt = alt_hi.p;
    if (n_keys > 1) {
      SB_TRY((sort_pairs<uint64_t, uint64_t>(tmp, klo, klo_alt, khi, khi_alt, n_keys, 0, 64, false, s)));
      SB_TRY((sort_pairs<uint64_t, uint64_t>(tmp, khi, khi_alt, klo, klo_alt, n_keys, 0, 64, false, s)));
    }
    if (klo != g->id_lo.p) SB_CUDA(cudaMemcpyAsync(g->id_lo.p, klo, n_keys * 8, cudaMemcpyDeviceToDevice, s));
    if (khi != g->id_hi.p) SB_CUDA(cudaMemcpyAsync(g->id_hi.p, khi, n_keys * 8, cudaMemcpyDeviceToDevice, s));
    if (has_max) {  // the all-ones id is the largest possible u128: it takes the last rank
      SB_CUDA(cudaMemsetAsync(g->id_lo.p + n_keys, 0xFF, 8, s));
      SB_CUDA(cudaMemsetAsync(g->id_hi.p + n_keys, 0xFF, 8, s));
    }
    SB_CUDA(cudaStreamSynchronize(s));
  }
  pt.mark("1c assign ranks");
  DevBuf<uint32_t> slot_val; SB_TRY(slot_val.alloc(cap));
  if (n_keys) {
    SB_LAUNCH(k_assign_ranks, div_up(n_keys, TPB), TPB, 0, s, g->id_lo.p, g->id_hi.p, n_keys, table.p, slot_val.p, cap - 1);
    SB_CHECK_LAUNCH();
  }

  pt.mark("2a map edges");
  // ---- 2. edges -> (to_rank<<32|from_rank), stable sort, unique_by first-wins, drop skipped ----
  DevBuf<uint64_t> keys_a, keys_b; SB_TRY(keys_a.alloc(n_edges)); SB_TRY(keys_b.alloc(n_edges));
  if (n_edges) {
    SB_LAUNCH(k_map_slots, div_up(n_edges, TPB), TPB, 0, s, slot_from.p, slot_to.p, n_edges, slot_val.p, (uint32_t)(N - 1), keys_a.p);
    SB_CHECK_LAUNCH();
  }
  SB_CUDA(cudaStreamSynchronize(s));
  slot_from.release(); slot_to.release();
  table.release(); slot_val.release();

  pt.mark("2b sort pairs + select");
  const int nb = bits_for(N);
  uint64_t *k = keys_a.p, *k_alt = keys_b.p; uint8_t *sk = skip_a.p, *sk_alt = skip_b.p;
  SB_TRY((sort_pairs<uint64_t, uint8_t>(tmp, k, k_alt, sk, sk_alt, n_edges, 0, 32 + nb, false, s)));
  SB_TRY(g->self_bm.alloc((N + 31) / 32 + 1));
  SB_CUDA(cudaMemsetAsync(g->self_bm.p, 0, ((N + 31) / 32 + 1) * 4, s));
  SB_LAUNCH(k_mark_keep, div_up(n_edges, TPB), TPB, 0, s, k, sk, n_edges, sk_alt, g->self_bm.p);
  SB_CHECK_LAUNCH();
  {
    size_t need = 0;
    SB_CUDA(cub::DeviceSelect::Flagged(nullptr, need, k, sk_alt, k_alt, ctr.p, (int64_t)n_edges, s));
    if (tmp.n < need) SB_TRY(tmp.alloc(need + 256));
    SB_CUDA(cub::DeviceSelect::Flagged(tmp.p, need, k, sk_alt, k_alt, ctr.p, (int64_t)n_edges, s));
    g_launches.fetch_add(2, std::memory_order_relaxed);
    SB_CUDA(cudaMemcpyAsync(h_ctr, ctr.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaStreamSynchronize(s));
  }
  const uint64_t E = h_ctr[0];
  g->E_kept = E;
  std::swap(k, k_alt);  // k = kept keys in rank space, sorted by (to, from)
  skip_a.release(); skip_b.release();

  pt.mark("3a degrees + node sort");
  // ---- 3. degree-sorted relabel + destination-major CSR ------------------------------------------
  DevBuf<uint32_t> deg_a, deg_b, val_b; SB_TRY(deg_a.alloc(N)); SB_TRY(deg_b.alloc(N)); SB_TRY(val_b.alloc(N));
  SB_CUDA(cudaMemsetAsync(deg_a.p, 0, N * 4, s));
  if (E) { SB_LAUNCH(k_degree_hi, div_up(E, TPB), TPB, 0, s, k, E, deg_a.p); SB_CHECK_LAUNCH(); }
  SB_LAUNCH(k_iota, div_up(N, TPB), TPB, 0, s, g->perm.p, N); SB_CHECK_LAUNCH();
  uint32_t *dk = deg_a.p, *dk_alt = deg_b.p, *pv = g->perm.p, *pv_alt = val_b.p;
  SB_TRY((sort_pairs<uint32_t, uint32_t>(tmp, dk, dk_alt, pv, pv_alt, N, 0, 32, true, s)));
  if (pv != g->perm.p) SB_CUDA(cudaMemcpyAsync(g->perm.p, pv, N * 4, cudaMemcpyDeviceToDevice, s));
  SB_LAUNCH(k_invert, div_up(N, TPB), TPB, 0, s, g->perm.p, N, g->inv.p); SB_CHECK_LAUNCH();
  // dk = in-degree by internal row, descending
  SB_TRY(exclusive_scan_u32(tmp, dk, g->row_ptr.p, N, s));
  {
    uint32_t e32 = (uint32_t)E;
    SB_CUDA(cudaMemcpyAsync(g->row_ptr.p + N, &e32, 4, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemsetAsync(ctr.p, 0, 8 * sizeof(unsigned long long), s));
    SB_LAUNCH(k_class_bounds, div_up(N, TPB), TPB, 0, s, dk, N, 0u, (uint32_t)QUAD_MAX_DEG, (uint32_t)CHUNK_EDGES, ctr.p);
    SB_CHECK_LAUNCH();
    SB_CUDA(cudaMemcpyAsync(h_ctr, ctr.p, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaStreamSynchronize(s));
  }
  const uint64_t n_pos = h_ctr[0], n_warp = h_ctr[1], n_multi = h_ctr[2];
  g->n_pos = n_pos;

  pt.mark("3b row permute (dst CSR)");
  // destination-major CSR in internal ids: the rows move as blocks instead of re-sorting every edge (see k_row_permute)
  DevBuf<uint32_t> col_full; SB_TRY(col_full.alloc(E));
  if (E) {
    DevBuf<uint32_t> rank_ptr; SB_TRY(rank_ptr.alloc(N + 1));
    SB_LAUNCH(k_offsets_from_sorted, div_up(E + 1, TPB), TPB, 0, s, k, E, N, rank_ptr.p); SB_CHECK_LAUNCH();
    SB_LAUNCH(k_row_permute, div_up(E, TPB), TPB, 0, s, k, E, rank_ptr.p, g->inv.p, g->row_ptr.p, col_full.p); SB_CHECK_LAUNCH();
    SB_CUDA(cudaStreamSynchronize(s));
  } else if (g->world == 1) {
    SB_TRY(g->fwd_ptr.alloc(N + 1));
    SB_CUDA(cudaMemsetAsync(g->fwd_ptr.p, 0, (N + 1) * 4, s));
    g->has_fwd = true;
  }
  keys_a.release(); keys_b.release();

  pt.mark("4 partition");
  // ---- 4. owned slice of the CSR + pull work partition --------------------------------------------
  // Sharded handles own destination rows INTERLEAVED in blocks of 32 (row block b belongs to rank b % world, see
  // owned_row() in hyperball.cu): in the degree-sorted order every rank then holds 1/world of every degree class,
  // which balances both the gather work and -- decisive on 8 GPUs -- the bytes each rank has to push to its peers
  // (a contiguous edge-balanced split left one rank owning 78 % of the rows and 9.7 GB of NVLink egress per
  // iteration).  Every rank keeps the full CSR and filters by ownership inside the kernels.
  g->E_local = E;
  g->col = std::move(col_full);
  if (g->world > 1 && N) {
    SB_CUDA(cudaMemsetAsync(ctr.p, 0, sizeof(unsigned long long), s));
    SB_LAUNCH(k_owned_edges, div_up(N, TPB), TPB, 0, s, g->row_ptr.p, N, (uint32_t)g->world, (uint32_t)g->rank, ctr.p);
    SB_CHECK_LAUNCH();
    SB_CUDA(cudaMemcpyAsync(h_ctr, ctr.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaStreamSynchronize(s));
    g->E_local = h_ctr[0];
  }
  g->warp_row_begin = 0; g->warp_row_end = n_warp;
  g->quad_row_begin = n_warp; g->quad_row_end = n_pos;
  {
    uint32_t rp[3] = {0, 0, 0};
    SB_CUDA(cudaMemcpyAsync(&rp[0], g->row_ptr.p + g->warp_row_begin, 4, cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaMemcpyAsync(&rp[1], g->row_ptr.p + g->warp_row_end, 4, cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaMemcpyAsync(&rp[2], g->row_ptr.p + g->quad_row_end, 4, cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaStreamSynchronize(s));
    g->E_warp = rp[1] - rp[0];
    g->E_quad = (g->quad_row_end > g->quad_row_begin) ? rp[2] - rp[1] : 0;
  }
  g->own_frac = 1.0;
  if (g->world > 1 && E) g->own_frac = (double)g->E_local / (double)E;   // share of every degree class this rank owns (interleaved blocks)
  const uint64_t nwr = g->warp_row_end - g->warp_row_begin;
  g->n_items = 0; g->n_multi_rows = 0; g->n_multi_items = 0;
  if (nwr) {
    DevBuf<uint32_t> nchunks; SB_TRY(nchunks.alloc(nwr + 1));
    SB_CUDA(cudaMemsetAsync(nchunks.p, 0, (nwr + 1) * 4, s));
    SB_LAUNCH(k_row_chunks, div_up(nwr, TPB), TPB, 0, s, g->row_ptr.p, g->warp_row_begin, nwr, CHUNK_EDGES, nchunks.p);
    SB_CHECK_LAUNCH();
    SB_TRY(g->item_start.alloc(nwr + 1));
    SB_TRY(exclusive_scan_u32(tmp, nchunks.p, g->item_start.p, nwr + 1, s));
    uint32_t total = 0, multi_items = 0;
    SB_CUDA(cudaMemcpyAsync(&total, g->item_start.p + nwr, 4, cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaMemcpyAsync(&multi_items, g->item_start.p + n_multi, 4, cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaStreamSynchronize(s));
    g->n_items = total; g->n_multi_rows = n_multi; g->n_multi_items = multi_items;
    SB_TRY(g->item_row.alloc(total));
    SB_LAUNCH(k_fill_items, div_up(total, TPB), TPB, 0, s, g->item_start.p, nwr, (uint64_t)total,
              (uint32_t)g->warp_row_begin, g->item_row.p);
    SB_CHECK_LAUNCH();
    SB_TRY(g->partial.alloc((size_t)std::max<uint64_t>(1, g->n_multi_items) * 4));
    SB_CUDA(cudaStreamSynchronize(s));
  }
  if (g->world > 1 && N) {
    // every rank holds the full CSR, so it derives the subscriber mask of every node itself (no exchange needed)
    pt.mark("5 subscriber masks");
    SB_TRY(g->sub_mask.alloc(N));
    SB_CUDA(cudaMemsetAsync(g->sub_mask.p, 0, N * 4, s));
    if (g->n_items) {
      SB_LAUNCH(k_sub_items, div_up(g->n_items * 32, TPB), TPB, 0, s, g->n_items, g->item_row.p, g->item_start.p,
                (uint32_t)g->warp_row_begin, g->row_ptr.p, g->col.p, CHUNK_EDGES, (uint32_t)g->world, g->sub_mask.p);
      SB_CHECK_LAUNCH();
    }
    if (g->quad_row_end > g->quad_row_begin) {
      SB_LAUNCH(k_sub_rows, div_up(g->quad_row_end - g->quad_row_begin, TPB), TPB, 0, s, g->quad_row_begin, g->quad_row_end,
                g->row_ptr.p, g->col.p, (uint32_t)g->world, g->sub_mask.p);
      SB_CHECK_LAUNCH();
    }
    g->n_owned_items = 0;
    if (g->n_items) {
      DevBuf<uint32_t> flag, pos;
      SB_TRY(flag.alloc(g->n_items + 1)); SB_TRY(pos.alloc(g->n_items + 1));
      SB_LAUNCH(k_item_owned_flag, div_up(g->n_items + 1, TPB), TPB, 0, s, g->n_items, g->item_row.p, (uint32_t)g->world, (uint32_t)g->rank, flag.p);
      SB_CHECK_LAUNCH();
      SB_TRY(exclusive_scan_u32(tmp, flag.p, pos.p, g->n_items + 1, s));
      uint32_t n_own = 0;
      SB_CUDA(cudaMemcpyAsync(&n_own, pos.p + g->n_items, 4, cudaMemcpyDeviceToHost, s));
      SB_CUDA(cudaStreamSynchronize(s));
      SB_TRY(g->owned_items.alloc((size_t)n_own + 1));
      SB_LAUNCH(k_item_owned_scatter, div_up(g->n_items, TPB), TPB, 0, s, g->n_items, flag.p, pos.p, g->owned_items.p);
      SB_CHECK_LAUNCH();
      SB_CUDA(cudaStreamSynchronize(s));
      g->n_owned_items = n_own;
    }
    SB_CUDA(cudaMemsetAsync(ctr.p, 0, sizeof(unsigned long long), s));
    SB_LAUNCH(k_sub_count, div_up(N, TPB), TPB, 0, s, g->sub_mask.p, N, (uint32_t)g->world, (uint32_t)g->rank, ctr.p);
    SB_CHECK_LAUNCH();
    SB_CUDA(cudaMemcpyAsync(h_ctr, ctr.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaStreamSynchronize(s));
    g->n_subscribed = h_ctr[0];
  }
  pt.mark(nullptr);
  SB_CUDA(cudaEventRecord(g->ev1, s));
  SB_CUDA(cudaStreamSynchronize(s));
  float ms = 0; cudaEventElapsedTime(&ms, g->ev0, g->ev1);
  g->stage_ms = ms;
  return SB200_OK;
}

int build_fwd_csr(sb200_graph* g) {
  if (g->has_fwd) return SB200_OK;
  cudaStream_t s = g->stream;
  const uint64_t N = g->N;
  // a sharded handle pushes only into the rows it owns: its source-major CSR holds the E_local edges whose
  // destination is owned (every rank resolves the whole frontier against its own slice)
  const uint64_t E = g->world == 1 ? g->E_kept : g->E_local;
  const int TPB = 256;
  SB_TRY(g->fwd_ptr.alloc(N + 1));
  if (E == 0) { SB_CUDA(cudaMemsetAsync(g->fwd_ptr.p, 0, (N + 1) * 4, s)); SB_CUDA(cudaStreamSynchronize(s)); g->has_fwd = true; return SB200_OK; }
  DevBuf<uint64_t> ka, kb; SB_TRY(ka.alloc(E)); SB_TRY(kb.alloc(E));
  if (g->world > 1) {
    DevBuf<uint32_t> deg, own_ptr; SB_TRY(deg.alloc(N + 1)); SB_TRY(own_ptr.alloc(N + 1));
    SB_LAUNCH(k_owned_deg, div_up(N + 1, TPB), TPB, 0, s, g->row_ptr.p, N, (uint32_t)g->world, (uint32_t)g->rank, deg.p);
    SB_CHECK_LAUNCH();
    SB_TRY(exclusive_scan_u32(g->cub_tmp, deg.p, own_ptr.p, N + 1, s));
    if (g->n_items) {
      SB_LAUNCH(k_fwd_keys_items_own, div_up(g->n_items * 32, TPB), TPB, 0, s, g->n_items, g->item_row.p, g->item_start.p,
                (uint32_t)g->warp_row_begin, g->row_ptr.p, own_ptr.p, g->col.p, CHUNK_EDGES, (uint32_t)g->world,
                (uint32_t)g->rank, ka.p);
      SB_CHECK_LAUNCH();
    }
    if (g->quad_row_end > g->quad_row_begin) {
      SB_LAUNCH(k_fwd_keys_rows_own, div_up(g->quad_row_end - g->quad_row_begin, TPB), TPB, 0, s, g->quad_row_begin,
                g->quad_row_end, g->row_ptr.p, own_ptr.p, g->col.p, (uint32_t)g->world, (uint32_t)g->rank, ka.p);
      SB_CHECK_LAUNCH();
    }
    SB_CUDA(cudaStreamSynchronize(s));  // deg / own_ptr go out of scope
  } else {
  if (g->n_items) {
    SB_LAUNCH(k_fwd_keys_items, div_up(g->n_items * 32, TPB), TPB, 0, s, g->n_items, g->item_row.p, g->item_start.p,
              (uint32_t)g->warp_row_begin, g->row_ptr.p, g->col.p, CHUNK_EDGES, ka.p);
    SB_CHECK_LAUNCH();
  }
  if (g->quad_row_end > g->quad_row_begin) {
    SB_LAUNCH(k_fwd_keys_rows, div_up(g->quad_row_end - g->quad_row_begin, TPB), TPB, 0, s, g->quad_row_begin, g->quad_row_end,
              g->row_ptr.p, g->col.p, ka.p);
    SB_CHECK_LAUNCH();
  }
  }
  uint64_t *a = ka.p, *b = kb.p;
  SB_TRY(sort_keys<uint64_t>(g->cub_tmp, a, b, E, 0, 32 + bits_for(N), s));
  SB_TRY(g->fwd_dst.alloc(E));
  SB_LAUNCH(k_lo32, div_up(E, TPB), TPB, 0, s, a, E, g->fwd_dst.p); SB_CHECK_LAUNCH();
  SB_LAUNCH(k_offsets_from_sorted, div_up(E + 1, TPB), TPB, 0, s, a, E, N, g->fwd_ptr.p); SB_CHECK_LAUNCH();
  SB_CUDA(cudaStreamSynchronize(s));
  g->cub_tmp.release();
  g->has_fwd = true;
  return SB200_OK;
}

}  // namespace sb200
