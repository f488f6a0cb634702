/* stract_b200.h -- C ABI of libstract_b200.so: H100-native (sm_90a) replacements for Stract's
 * two data-parallel ranking hot paths.  This is the drop-in boundary a Rust `extern "C"` block
 * (see INTEGRATION.md) binds; every entry point cites the reference interface it replaces
 * (paths relative to the root of the Stract repository).
 *
 * Conventions
 *   - plain pointers + sizes; the caller owns every buffer; nothing is retained after return
 *     except by the *_create calls, which COPY their inputs into device memory (HBM);
 *   - input pointers may be host OR device pointers (detected with cudaPointerGetAttributes);
 *     output pointers are host pointers unless a function says otherwise;
 *   - every function returns 0 on success or a negative SB200_E* code; the message of the last
 *     error on the calling thread is available from sb200_last_error(); nothing unwinds or
 *     aborts across the boundary (reference: crate::Result / anyhow::Result);
 *   - handles are not thread-safe: one caller at a time per handle (each owns a CUDA stream);
 *     distinct handles may be used concurrently (reference: Collector: Sync+Send used from one
 *     thread per segment, crates/tantivy/src/collector/mod.rs:133-152).
 */
#ifndef STRACT_B200_H
#define STRACT_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define SB200_API __attribute__((visibility("default")))
#else
#define SB200_API
#endif

#define SB200_OK 0
#define SB200_EINVAL (-1)   /* bad argument */
#define SB200_ECUDA (-2)    /* CUDA runtime error (message has the cudaError string) */
#define SB200_ENOMEM (-3)   /* device or host allocation failed */
#define SB200_ERANGE (-4)   /* input exceeds a documented limit (e.g. > 2^32-2 nodes) */
#define SB200_ESTATE (-5)   /* call sequence error (e.g. result before run) */
#define SB200_EFORMAT (-6)  /* malformed posting bytes */

SB200_API const char* sb200_last_error(void);
/* library version, number of kernels launched by this process so far (bench evidence) */
SB200_API const char* sb200_version(void);
SB200_API uint64_t sb200_kernel_launch_count(void);

/* ===========================================================================================
 * Path 1 -- webgraph harmonic centrality (HyperBall)
 *   replaces  HarmonicCentrality::calculate(&Webgraph)  crates/core/src/webgraph/centrality/harmonic.rs:289-311
 *   fed by    Webgraph::host_edges()/host_nodes()        crates/core/src/webgraph/mod.rs:157-194
 *   and, with world_size > 1, the whole AMPC round loop   crates/core/src/entrypoint/ampc/harmonic_centrality/
 * =========================================================================================== */
typedef struct sb200_graph sb200_graph;

/* Drain of `graph.host_edges()` as SoA: edge i is (from = from_hi[i]<<64|from_lo[i]) ->
 * (to = ...), rel_flags[i] = RelFlags bits (crates/core/src/webpage/html/links.rs:114-141).
 * Semantics reproduced from the reference iterator (crates/core/src/webgraph/store.rs:297-357):
 *   - nodes  = every endpoint of every edge, including skipped ones;
 *   - edges are de-duplicated on (from,to), the FIRST occurrence's rel_flags decide;
 *   - an edge is ignored by the iteration iff rel_flags & skipped_rel_mask != 0
 *     (SKIPPED_REL, harmonic.rs:36-49; pass SB200_SKIPPED_REL_DEFAULT for the reference's mask).
 * The library relabels u128 ids to dense u32 indices, builds a destination-major CSR (and a
 * source-major one for small frontiers) in HBM and keeps 2 x N x 64 B of HyperLogLog registers.
 *
 * Sharding (reference: one CentralityJob{shard} per worker, mapper.rs:356-369): with world_size > 1
 * every rank must be given the SAME full edge stream; it keeps the full CSR and register array and
 * OWNS the destination rows of every world_size-th 32-row block of the internal (degree-sorted)
 * order (row block b -> rank b % world_size), so all ranks hold an equal share of every degree class. */
#define SB200_SKIPPED_REL_DEFAULT 0x6FED00ull /* bits 8,10,11,13-19,21,22 */

SB200_API int sb200_graph_create(const uint64_t* from_lo, const uint64_t* from_hi, const uint64_t* to_lo,
                       const uint64_t* to_hi, const uint64_t* rel_flags, uint64_t n_edges,
                       uint64_t skipped_rel_mask, int device, int rank, int world_size,
                       sb200_graph** out);
SB200_API void sb200_graph_destroy(sb200_graph* g);

typedef struct {
  uint64_t n_nodes;        /* |host_nodes()| */
  uint64_t n_edges_input;  /* edges handed to create */
  uint64_t n_edges_kept;   /* unique, non-skipped, non-self-loop edges in the CSR (all ranks) */
  uint64_t n_edges_local;  /* ... of which this rank owns (== kept when world_size == 1) */
  uint64_t row_begin, row_end; /* always 0 and n_nodes: rows are owned in interleaved 32-row blocks (sb200_graph_ownership) */
  uint64_t hbm_bytes;      /* device memory held by the handle */
  double stage_ms;         /* device time spent in create (relabel + CSR build) */
} sb200_graph_info;
SB200_API int sb200_graph_get_info(const sb200_graph* g, sb200_graph_info* info);

/* Tuning/debug hook: which kernel family an iteration uses.  An iteration whose frontier covers
 * >= dense_frac of the edges gathers every in-neighbour (dense pull); one whose frontier out-edges
 * are <= E/push_div pushes from the frontier (the reference's small-frontier branch,
 * harmonic.rs:244-252); otherwise frontier-filtered pull.  force_mode 0/1/2 pins a family (-1 = auto).
 * All three compute the same result; negative dense_frac / non-positive push_div keep the current value. */
SB200_API int sb200_hyperball_set_policy(sb200_graph* g, double dense_frac, double push_div, int force_mode);

/* (Re)initialise the iteration state: counters seeded with each node's own id (harmonic.rs:53-73),
 * centralities zero, frontier = all nodes (harmonic.rs:221-225). create() leaves the handle reset. */
SB200_API int sb200_hyperball_reset(sb200_graph* g);

typedef struct {
  uint32_t t;              /* iteration index just executed (0-based) */
  uint32_t mode;           /* 0 dense pull, 1 frontier-filtered pull, 2 push from frontier */
  uint64_t n_changed;      /* nodes whose registers changed (this rank's rows when sharded) */
  uint64_t edges_active;   /* edges whose source was in the frontier (0 if not tracked) */
  float ms;                /* device time of the iteration */
} sb200_iter_stats;

/* One synchronous iteration new[v] = max(old[v], max_{u->v} old[u]) + centrality update
 * (update_all_counters / update_changed_counters + update_centralities + Counters::step,
 * harmonic.rs:75-176,210-212).  With world_size > 1 the caller must exchange the owned
 * register rows between ranks after each step (see sb200_hyperball_exchange_*). */
SB200_API int sb200_hyperball_step(sb200_graph* g, sb200_iter_stats* stats);

/* calculate_centrality (harmonic.rs:215-287): iterate until an iteration changes nothing
 * (max_iters == 0) or at most max_iters iterations.  Single-rank handles only. */
SB200_API int sb200_hyperball_run(sb200_graph* g, uint32_t max_iters, uint32_t* iters_done,
                        sb200_iter_stats* per_iter /* nullable, capacity cap */, uint32_t cap);

/* Device time (CUDA events on the handle's stream) of the last sb200_hyperball_run call. */
SB200_API int sb200_hyperball_last_run_ms(sb200_graph* g, float* ms);

/* Per-kernel-family device timing, measured with CUDA events on the stream the kernels are launched
 * on; `alg_bytes` is the algorithmic (not measured) HBM traffic of the family's launches: the
 * numerator of the roofline bench.py reports (DESIGN.md states the per-unit figures). */
typedef struct { char name[32]; uint64_t launches; double ms; double alg_bytes; } sb200_kernel_prof;
SB200_API int sb200_hyperball_set_profiling(sb200_graph* g, int on); /* also clears the accumulators */
SB200_API int sb200_hyperball_get_profile(sb200_graph* g, sb200_kernel_prof* out, uint32_t cap, uint32_t* n);

/* HarmonicCentrality::iter() (harmonic.rs:300-302): ascending u128 id, only centrality > 0,
 * already divided by (N-1) (normalize_centralities, harmonic.rs:178-195).  Call with
 * centrality == NULL to get the length.  Sharded handles return only their owned nodes. */
SB200_API int sb200_hyperball_result(sb200_graph* g, uint64_t* id_lo, uint64_t* id_hi, double* centrality,
                           uint64_t cap, uint64_t* len);

/* Rank assignment, the step right behind the centrality computation (SURVEY 8(f) rank 1): store_harmonic sorts
 * (Reverse(SortableFloat(centrality)), node_id) and writes the position as `harmonic_rank`
 * (crates/core/src/webgraph/centrality/mod.rs:88-108); top_nodes takes the k largest (centrality, node_id) pairs
 * (mod.rs:17-37).  Output: the nodes with centrality > 0 ordered by centrality descending (f64 total order), ties by
 * node id ascending (ties_desc == 0: entry i has harmonic rank i) or descending (ties_desc != 0: top_nodes' order);
 * at most `cap` leading entries are written, *len = number of ranked nodes.  Single-rank handles only. */
SB200_API int sb200_hyperball_ranked(sb200_graph* g, int ties_desc, uint64_t* id_lo, uint64_t* id_hi, double* centrality,
                                     uint64_t cap, uint64_t* len);

/* Parity/debug hooks: state of nodes [first, first+count) in ascending-u128-id (rank) order. */
SB200_API int sb200_hyperball_registers(sb200_graph* g, uint64_t first, uint64_t count, uint8_t* out /* count*64 */);
SB200_API int sb200_hyperball_kahan(sb200_graph* g, uint64_t first, uint64_t count, double* sum, double* err);
SB200_API int sb200_graph_node_ids(sb200_graph* g, uint64_t first, uint64_t count, uint64_t* id_lo, uint64_t* id_hi);

/* Multi-GPU exchange hooks, collective variant.  The DHT upsert `HyperLogLog64Upsert` is an
 * elementwise max (crates/core/src/ampc/dht/upsert.rs:66-83); registers only grow and every row has one
 * owner, so after a step the caller merges the replicas with exactly that operator:
 *   regs      : the full N x 64 B "current" register array (device pointer, valid until the next step):
 *               ncclAllReduce(ncclUint8, ncclMax) in place (torch: all_reduce(op=MAX) on a uint8 view);
 *   frontier  : N-bit changed bitmap; each 32-bit word has a single owner (ownership is in 32-row blocks)
 *               and non-owners hold 0, so the same byte-wise max all-reduce yields the union;
 * then sums the per-rank changed counts and calls sb200_hyperball_exchange_done.
 * sb200_graph_row_ranges is kept for ABI compatibility and returns [0, ..., 0, N]. */
SB200_API int sb200_hyperball_exchange_ptrs(sb200_graph* g, void** regs, uint64_t* regs_bytes,
                                  void** frontier_words, uint64_t* frontier_bytes);
SB200_API int sb200_graph_row_ranges(sb200_graph* g, uint64_t* begins /* world_size+1 */);
/* Fused exchange (one process per GPU on one NVLink/NVSwitch box): every rank exports one blob -- CUDA IPC handles of
 * its two register arrays, two bitmaps and its sync page, plus its rank -- imports the blobs of all other ranks (any
 * order) and enables p2p.  From then on a step stores every produced row directly into the peers' replicas from inside
 * the pull kernels (st.global on peer pointers) and copies its owned changed-bitmap words to them, so no all-gather is
 * needed.  A row is stored only into the replicas of the ranks that gather it (subscriber mask = the owners of the
 * node's out-neighbours, derived from the CSR at create): a replica is authoritative for the rows its rank owns or
 * reads, the rest keep their initial value (sb200_graph_ownership names both sets).
 *   - sb200_hyperball_run_sharded runs the whole round loop (the AMPC coordinator's, crates/core/src/ampc/
 *     coordinator.rs:151-213, Meta.round_had_changes = the summed changed count): all ranks call it together; between
 *     iterations they meet in a device-side barrier over the mapped sync pages that also sums the changed counts --
 *     no host collective, no NCCL.  Returns SB200_ESTATE if a peer does not arrive within 20 s.
 *   - stepping by hand (sb200_hyperball_step) stays possible: the caller then supplies a barrier plus the sum of the
 *     per-rank changed counts between steps (one small all-reduce does both) and sb200_hyperball_exchange_done;
 *     a barrier is also required after create/reset before the first step. */
#define SB200_IPC_HANDLE_BYTES 64
#define SB200_IPC_BLOB_BYTES 384 /* 5 handles + {rank, world_size} as u32 + padding */
SB200_API int sb200_hyperball_ipc_export(sb200_graph* g, uint8_t* out /* SB200_IPC_BLOB_BYTES */);
SB200_API int sb200_hyperball_ipc_import(sb200_graph* g, const uint8_t* blob /* one peer's blob */);
SB200_API int sb200_hyperball_p2p_enable(sb200_graph* g, int on);
SB200_API int sb200_hyperball_run_sharded(sb200_graph* g, uint32_t max_iters, uint32_t* iters_done,
                                          sb200_iter_stats* per_iter /* nullable, capacity cap */, uint32_t cap);

/* The single-process form (one thread drives n handles: the n GPUs of one box, or several ranks on one GPU):
 * handles[i] must have been created with rank i / world_size n from the same edge stream.  group_link enables peer
 * access between the devices and wires every handle's publish targets to the other handles' arrays by address;
 * group_run is the round loop: each round launches the iteration on every handle, then waits for all of them and sums
 * the changed counts on the host.  per_iter (nullable) is an [n][cap] array. */
SB200_API int sb200_hyperball_group_link(sb200_graph** handles, int n);
SB200_API int sb200_hyperball_group_run(sb200_graph** handles, int n, uint32_t max_iters, uint32_t* iters_done,
                                        sb200_iter_stats* per_iter, uint32_t cap);

/* Per node, in ascending-id order: owned[i] = 1 iff this rank owns the node's row; subscribers[i] = bit mask of the ranks
 * whose replica receives the row (all ranks when the subscriber filter is off).  Either output may be NULL. */
SB200_API int sb200_graph_ownership(sb200_graph* g, uint8_t* owned, uint32_t* subscribers);

/* The same fused exchange over caller-owned memory, addressed directly instead of through CUDA IPC.  Meant for
 * "symmetric" memory that is bound to an NVSwitch multicast object on every rank (cuMemCreate +
 * cuMulticastBindMem; torch.distributed._symmetric_memory does exactly that):
 *   1. sb200_hyperball_state_bytes  -> sizes of one register array / one bitmap for this graph;
 *   2. the caller allocates 2 + 2 such buffers (register arrays 64-byte aligned) and hands their LOCAL mappings to
 *      sb200_hyperball_bind_state right after create: the handle drops its own arrays, uses these (never frees
 *      them; they must outlive the handle) and re-initialises the HyperBall state;
 *   3. sb200_hyperball_set_publish_targets names where produced rows / bitmap words are stored in addition to the
 *      local replica: either world_size-1 unicast peer mappings IN RANK ORDER (own rank left out; the subscriber
 *      filter applies), or ONE multicast mapping (n_targets = 1; reaches every replica, filter off) -- a store
 *      to a multicast address is replicated by the switch into every rank's replica, so a produced row leaves the
 *      GPU once instead of world_size-1 times.  n_targets = 0 switches the fused exchange off.
 * Inter-step protocol as above (barrier + changed-count all-reduce, then sb200_hyperball_exchange_done). */
SB200_API int sb200_hyperball_state_bytes(sb200_graph* g, uint64_t* regs_bytes, uint64_t* bitmap_bytes);
SB200_API int sb200_hyperball_bind_state(sb200_graph* g, void* regs0, void* regs1, void* bitmap0, void* bitmap1);
SB200_API int sb200_hyperball_set_publish_targets(sb200_graph* g, int n_targets, const uint64_t* regs0,
                                                  const uint64_t* regs1, const uint64_t* bitmap0, const uint64_t* bitmap1);

/* after the exchange: tell the library the global changed count so every rank picks the same mode */
SB200_API int sb200_hyperball_exchange_done(sb200_graph* g, uint64_t global_n_changed);

/* ---- other graph kernels over the resident CSR (SURVEY 8(f) rank 4) --------------------------------------------------
 * All edge costs are 1, so the reference's dijkstra_multi (crates/core/src/webgraph/shortest_path.rs:57-105) is a
 * breadth-first search; up to 64 searches run bit-parallel over the CSR the handle already holds.  Single-rank handles.
 * The edge set is the handle's (unique, non-self-loop edges that pass skipped_rel_mask): create the handle with
 * skipped_rel_mask = 0 for searches over every link, as ForwardlinksQuery / BacklinksQuery see them.
 *
 * sb200_graph_distances: raw_distances / raw_distances_with_max (forward, reversed = 0) and raw_reversed_distances(_with_max)
 * (shortest_path.rs:122-214).  Source i belongs to search src_group[i] (NULL: its own search); a search with several
 * sources reports the distance to the nearest one (dijkstra_multi's `sources` slice).  dist_out is [n_groups][n_nodes] in
 * ascending-id order, 255 = not reached.  max_dist = 0: unbounded; otherwise the reference's cut-off is reproduced: it
 * returns when it POPS a node with cost > max_dist, so nodes at distance max_dist + 1 are still reported. */
SB200_API int sb200_graph_distances(sb200_graph* g, const uint64_t* src_lo, const uint64_t* src_hi, const uint32_t* src_group,
                                    uint32_t n_sources, uint32_t n_groups, uint32_t max_dist, int reversed, uint8_t* dist_out);
/* ApproxHarmonic::build (crates/core/src/webgraph/centrality/approx_harmonic.rs:40-88) for a caller-chosen sample (the
 * reference draws random page nodes with outgoing links; ceil(log2(n) / 0.3^2) of them): one forward search with
 * max_dist (7 in the reference) per sample; every reached target at distance d >= 1 receives
 * (1.0 / d as f32) * (num_nodes as f32 / (n_sources as f32 * (num_nodes as f32 - 1.0))).  num_nodes is the reference's
 * HyperLogLog<2048> estimate of the node count (0: the exact count).  The reference accumulates the f32 terms in a
 * DashMap from a rayon pool, i.e. in no defined order; here the same f32 terms are summed in f64.  Output: the nodes that
 * were reached, ascending id; call with centrality == NULL for the length. */
SB200_API int sb200_approx_harmonic(sb200_graph* g, const uint64_t* src_lo, const uint64_t* src_hi, uint32_t n_sources,
                                    uint32_t max_dist, uint64_t num_nodes, uint64_t* id_lo, uint64_t* id_hi, double* centrality,
                                    uint64_t cap, uint64_t* len);
/* Betweenness::calculate (crates/core/src/webgraph/centrality/betweenness.rs:29-146) for the caller's sources, in the given
 * order (the reference takes the first 100 000 of an FxHashSet): Brandes' algorithm, one forward search per source over
 * every kept link, sigma counted in i32 that wraps like the reference's release build, then
 *     delta[v] = delta[v] + (sigma[v] as f64 / sigma[w] as f64) * (1.0 + delta[w])
 * over v's successors w on the shortest-path DAG in ascending node id, and centrality[w] += delta[w] (w != source) in source
 * order; the result is centrality / (n * (n - 1.0)), n = n_sources (n == 1 divides by zero, as in the reference).
 * Output: every source and every node a source reaches, ascending id, at most n_nodes entries; max_dist = the largest
 * distance of any search.  Refused: a source id that is not a node or repeats an earlier one, cap < n_nodes (SB200_EINVAL),
 * a distance of 255 or more (SB200_ERANGE: distances are u8).  Single-rank handles. */
SB200_API int sb200_betweenness(sb200_graph* g, const uint64_t* src_lo, const uint64_t* src_hi, uint32_t n_sources, uint64_t* id_lo,
                                uint64_t* id_hi, double* centrality, uint64_t cap, uint64_t* len, uint32_t* max_dist);

/* Inbound similarity (crates/core/src/ranking/inbound_similarity.rs:71-119 over bitvec_similarity.rs:130-185): for every
 * candidate node, Scorer::score against the liked / disliked nodes:
 *     s = |disliked| + (sum_liked sim - sum_disliked sim),  s / max(|liked|, 1) if normalized,  max(s, 0)
 *     sim(a, b) = |in(a) ∩ in(b)| / (sqrt|in(a)| * sqrt|in(b)|), 0 if either set is empty or if the reference's 16 x 64-bit
 *                 bloom pre-filter over the low 64 id bits says popcount(A & B) / max(ones) < 0.25 (false negatives included);
 *     a liked / disliked node compared with itself scores self_score (1.0 in the reference until set_self_score).
 * in(v) = the unique sources of v's links in the handle's edge set, including v itself if it links to itself.  Ids that are
 * not nodes of the graph have an empty set.  Single-rank handles.
 * The reference fills the sets from `HostBacklinksQuery(...).with_limit(512)` and then drops NOFOLLOW edges
 * (crates/core/src/searcher/api/mod.rs:199-214): stage the handle with skipped_rel_mask = NOFOLLOW for the filter; the 512-edge
 * limit (the store's own top-docs order) is the caller's to apply to the edge stream -- the handle does not truncate. */
SB200_API int sb200_inbound_similarity(sb200_graph* g, const uint64_t* liked_lo, const uint64_t* liked_hi, uint32_t n_liked,
                                       const uint64_t* disliked_lo, const uint64_t* disliked_hi, uint32_t n_disliked,
                                       const uint64_t* cand_lo, const uint64_t* cand_hi, uint32_t n_cand, int normalized,
                                       double self_score, double* scores);

/* Tuning switches of one handle: "quad_side_ctas" (CTAs per SM of the short-row kernel on the side stream of the fused
 * exchange, 0 = one stream; default 2 with up to 4 ranks or one multicast target, else 0), "owned_items" (0 / 1: launch the
 * long-row kernel over the owned work items only; default 1), "publish_all" (0 / 1: store produced rows into every peer, no
 * subscriber filter; default 0), "l2_window_mb" (size of the persisting L2 window over the head of the register array, 0..1024 MiB,
 * capped by the device; 0 = no window; default 16), "l1_hub_kb" (L1 budget of the pulls' hub sources, 0..2^30 KiB: the first
 * kb * 1024 / 64 rows are gathered through L1 and every other source around it; 0 = no gather through L1, at least
 * N * 64 / 1024 = every gather through L1; default: every gather through L1).  All ranks of a sharded computation must use the same "publish_all".
 * Not while an iteration is in flight. */
SB200_API int sb200_hyperball_set_option(sb200_graph* g, const char* name, double value);

/* Device-memory arena diagnostics.  With SB200_ARENA=1 in the environment, staging temporaries, the CSR and the
 * state of single-rank handles are sub-allocated from large slabs that are kept for the life of the process
 * (deterministic, no driver call per allocation once warm) instead of the driver's stream-ordered pool.
 * sb200_arena_trim returns empty slabs to the driver; sb200_arena_selftest runs the allocator's randomised
 * invariant test over host memory (no GPU needed) and returns 0 on success. */
SB200_API int sb200_arena_stats(int device, uint64_t* reserved_bytes, uint64_t* in_use_bytes, uint64_t* peak_bytes,
                                uint64_t* n_slabs);
SB200_API int sb200_arena_trim(int device);
/* returns the memory cached for staging (the stream-ordered pool and empty arena slabs) to the driver */
SB200_API int sb200_release_cached_memory(int device);
SB200_API int sb200_arena_selftest(uint64_t seed, uint32_t ops);

/* ===========================================================================================
 * Path 2 -- BM25 posting-list scoring + top-k   (declared in stract_b200_bm25.h)
 * =========================================================================================== */

#ifdef __cplusplus
}
#endif
#endif
