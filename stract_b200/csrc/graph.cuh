// graph.cuh -- the sb200_graph handle: HBM layout of the host webgraph + HyperBall state.
//
// HBM layout (N nodes, E kept edges; "internal" node order = in-degree descending, so rows of
// similar length are adjacent and the degree classes are contiguous row ranges):
//   id_lo,id_hi  [N] u64      node ids ascending (rank order)          16 B/node
//   perm         [N] u32      internal -> rank;  inv [N] u32 rank -> internal
//   row_ptr      [N+1] u32    destination-major CSR offsets (internal) 4 B/node
//   col          [E_local] u32 source (internal) of every kept in-edge 4 B/edge
//   fwd_ptr/fwd_dst           source-major CSR for small frontiers     4 B/edge + 4 B/node
//   regs[2]      [N][64] u8   HyperLogLog<64> registers, ping-pong     128 B/node
//   seed         [N] u16      the one non-zero register of every reset counter, j | p << 8 (iteration 0 reads these)  2 B/node
//   bm[2]        [N/32] u32   changed bitmaps (previous / current)     2 bit/node
//   size_cache   [N] u64      size(old[v])                             8 B/node
//   kahan_sum/err[N] f64      KahanSum per node                        16 B/node
#pragma once
#include "common.cuh"

#include <vector>

namespace sb200 {
constexpr int MAX_PEERS = 15;
// publish targets of a sharded handle, by value in the kernel parameters.  `sub` (nullable) is the subscriber mask
// of every row: bit r is set iff rank r has an in-edge from that node, i.e. ever reads its row; with it a produced
// row is stored only into the replicas that will gather it (prank[p] = rank behind target p).
struct PeerOut { uint4* newr[MAX_PEERS]; uint32_t* bmc[MAX_PEERS]; const uint32_t* sub; int n; uint32_t world, rank; uint8_t prank[MAX_PEERS + 1]; };
// device-side barrier + changed-count sum between the ranks of one box (k_barrier_count): every rank owns a page of
// 2 x 64 slots (epoch parity x writer rank) that all peers map
constexpr int SYNC_SLOTS = 128;
struct SyncView { unsigned long long* local; unsigned long long* peer[MAX_PEERS]; int n; uint32_t world, rank; };
}

struct sb200_graph {
  int device = 0, rank = 0, world = 1;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  uint64_t N = 0, E_in = 0, E_kept = 0, E_local = 0;
  uint64_t n_pos = 0;  // rows [0, n_pos) have in-degree > 0 (globally)
  bool has_fwd = false;
  int reuse = 0;  // explicit resets: the source-major CSR (push branch) is only built once a handle is reused
  double stage_ms = 0;

  sb200::DevBuf<uint64_t> id_lo, id_hi;
  sb200::DevBuf<uint32_t> perm, inv;
  sb200::DevBuf<uint32_t> self_bm;  // [N/32] in RANK order: the node has a kept link to itself (not in the CSR: a no-op for HyperBall)
  sb200::DevBuf<uint32_t> row_ptr, col;
  sb200::DevBuf<uint32_t> fwd_ptr, fwd_dst;

  // pull work partition (every row; a sharded handle skips the rows it does not own inside the kernels)
  uint64_t warp_row_begin = 0, warp_row_end = 0;  // rows with deg > QUAD_MAX_DEG: warp-per-chunk
  uint64_t quad_row_begin = 0, quad_row_end = 0;  // rows with 0 < deg <= QUAD_MAX_DEG: quad-per-row
  uint64_t n_items = 0;                           // chunks of the warp rows
  uint64_t n_multi_rows = 0;                      // leading warp rows that span > 1 chunk
  sb200::DevBuf<uint32_t> owned_items;            // sharded: ascending ids of the items whose row this rank owns
  uint64_t n_owned_items = 0;
  sb200::DevBuf<uint32_t> item_row, item_start;   // item -> row ; row(-warp_row_begin) -> first item
  sb200::DevBuf<uint4> partial;                   // [n_multi_items][4] chunk partial registers
  uint64_t n_multi_items = 0;

  // iteration state
  sb200::DevBuf<uint8_t> regs[2];
  sb200::DevBuf<uint16_t> seed;   // written by hb_reset with the registers; every rank of a sharded handle holds all N
  sb200::DevBuf<uint32_t> bm[2];
  sb200::DevBuf<uint64_t> size_cache;
  sb200::DevBuf<double> kahan_sum, kahan_err;
  sb200::DevBuf<uint32_t> frontier_list, frontier_off;  // push mode scratch: sources + their first fwd_dst index, slot offsets
  sb200::DevBuf<unsigned long long> frontier_scan;       // push mode scratch: per bitmap word (sources << 32 | slots), + its scan
  sb200::DevBuf<uint8_t> cub_tmp;
  sb200::DevBuf<unsigned long long> counters;  // [0] n_changed [1] frontier out-edges [2..] scratch
  unsigned long long* h_counters = nullptr;    // pinned mirror
  int cur = 0;      // regs[cur] = "old"
  int bcur = 0;     // bm[bcur] = changed in the previous iteration
  uint32_t t = 0;
  bool has_changes = true;
  uint64_t n_changed_prev = 0, frontier_edges_prev = 0;
  bool exchange_pending = false;
  // fused multi-GPU exchange over peer memory (CUDA IPC): replicas of regs[2]/bm[2] on the other ranks
  int n_peers = 0;
  bool p2p = false;
  bool peers_ipc = true;  // peer mappings came from cudaIpcOpenMemHandle (closed at destroy); false: caller-owned addresses
  void* peer_regs[2][sb200::MAX_PEERS] = {{nullptr}};
  void* peer_bm[2][sb200::MAX_PEERS] = {{nullptr}};
  int peer_rank[sb200::MAX_PEERS] = {0};   // rank behind publish target p
  bool publish_all = false;                // one multicast target / set_option("publish_all"): no subscriber filtering
  sb200::DevBuf<uint32_t> sub_mask;        // [N] subscriber mask per row (internal order), sharded handles only
  uint64_t n_subscribed = 0;               // sum over owned rows of the number of remote subscribers (profile: NVLink rows per dense iteration)
  // device-side inter-rank barrier (sb200_hyperball_run_sharded)
  sb200::DevBuf<unsigned long long> sync_page;
  void* peer_sync[sb200::MAX_PEERS] = {nullptr};
  uint64_t sync_epoch = 0;
  bool step_in_flight = false, step_with_barrier = false;
  int step_mode = 0;
  double dense_frac = 0.35, push_div = 48.0;  // mode policy (see hb_step)
  int force_mode = -1;
  uint64_t l2_window_bytes = 0;  // persisting-L2 access window over the hot prefix of the `old` register array (hb_alloc_state)
  // L1 budget of the pulls' hub sources: the first l1_hub_bytes / 64 rows are gathered through L1 with evict_last, all
  // others around it (hyperball.cu, launch_pull; set_option "l1_hub_kb").  Default: every row (no budget below that was
  // faster at C2, DESIGN section 6)
  uint64_t l1_hub_bytes = UINT64_MAX;

  // optional per-kernel-family device timing (bench evidence; CUDA events on this handle's stream)
  enum { F_PULL_WARP_DENSE, F_PULL_QUAD_DENSE, F_PULL_WARP_FRONT, F_PULL_QUAD_FRONT, F_PULL_MERGE, F_PUSH, F_FINALIZE,
         F_PULL_WARP_SEED, F_PULL_QUAD_SEED, F_COUNT };
  bool profiling = false;
  uint64_t prof_launches[F_COUNT] = {0};
  double prof_ms[F_COUNT] = {0}, prof_bytes[F_COUNT] = {0};
  cudaEvent_t prof_ev[F_COUNT][2] = {{nullptr}};
  // fused exchange: the short-row kernel runs on a second stream beside the long-row kernel (hyperball.cu, launch_pull)
  int sm_count = 0;
  int opt_side_ctas = -1;    // -1: the default, chosen at first use (sb200_hyperball_set_option)
  int opt_owned_list = 1;    // k_pull_warp over the owned work items only (sb200_hyperball_set_option)
  cudaStream_t side_stream = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr, side_prof[2] = {nullptr, nullptr};
  bool side_prof_used = false;
  int side_prof_family = 0;
  bool prof_used[F_COUNT] = {false};
  double prof_step_bytes[F_COUNT] = {0};
  uint64_t E_warp = 0, E_quad = 0;   // edges of the warp-class / quad-class rows
  double own_frac = 1.0;             // sharded handles: fraction of the rows / edges of every class this rank owns
  cudaEvent_t ev_run0 = nullptr, ev_run1 = nullptr;
  float last_run_ms = 0;

  uint64_t hbm_bytes() const;
};

namespace sb200 {
constexpr int QUAD_MAX_DEG = 32;   // rows up to this in-degree: 4 lanes per row
constexpr int CHUNK_EDGES = 1024;  // longer rows are cut into warp-sized work items of this many edges

// source-major CSR from the resident destination-major one (lazy: see sb200_graph::reuse)
int build_fwd_csr(sb200_graph* g);
int stage_graph(sb200_graph* g, const uint64_t* from_lo, const uint64_t* from_hi, const uint64_t* to_lo,
                const uint64_t* to_hi, const uint64_t* rel, uint64_t n_edges, uint64_t mask);
__global__ void k_offsets_from_sorted(const uint64_t* keys, uint64_t n, uint64_t n_rows, uint32_t* ptr);

// bit-parallel searches (graph_bfs.cu), shared with the betweenness passes (graph_betweenness.cu)
struct BfsState {
  DevBuf<unsigned long long> frontier, next, visited, any;
  DevBuf<uint32_t> seed_rank, seed_bit;
};
// allocates the search words of `st` and maps the source ids to ranks (0xFFFFFFFF: not a node); single-rank handles
int bfs_prepare(sb200_graph* g, BfsState& st, const uint64_t* src_lo, const uint64_t* src_hi, uint32_t n_sources, std::vector<uint32_t>& ranks);
__global__ void k_bfs_seed(const uint32_t* seed_rank, const uint32_t* seed_bit, uint32_t n, const uint32_t* inv,
                           unsigned long long* frontier, unsigned long long* visited);
__global__ void __launch_bounds__(256) k_bfs_pull_items(uint64_t n_items, const uint32_t* item_row, const uint32_t* item_start,
    uint32_t warp_row_begin, const uint32_t* row_ptr, const uint32_t* col, const unsigned long long* frontier, unsigned long long* next);
__global__ void k_bfs_pull_rows(uint64_t row_begin, uint64_t row_end, const uint32_t* row_ptr, const uint32_t* col,
                                const unsigned long long* frontier, unsigned long long* next);
__global__ void k_bfs_commit(uint64_t N, const uint32_t* perm, unsigned long long* next, unsigned long long* visited,
                             unsigned long long* frontier, uint32_t level, uint8_t* dist_out, uint32_t n_bits, double* cent, double term,
                             unsigned long long* any);
__global__ void k_ah_scatter(const uint32_t* flag, const uint32_t* pos, const double* val, const uint64_t* id_lo, const uint64_t* id_hi,
                             uint64_t N, uint64_t cap, uint64_t* out_lo, uint64_t* out_hi, double* out_c);
}  // namespace sb200
