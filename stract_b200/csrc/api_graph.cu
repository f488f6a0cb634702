// api_graph.cu -- C ABI of path 1 (see include/stract_b200.h) + process-wide error/launch accounting.
#include "graph.cuh"

#include <algorithm>
#include <vector>

namespace sb200 {
static thread_local char t_err[1024] = "";
std::atomic<uint64_t> g_launches{0};
thread_local cudaStream_t t_pool_stream = nullptr;
void set_error(const char* fmt, ...) {
  va_list ap; va_start(ap, fmt);
  vsnprintf(t_err, sizeof(t_err), fmt, ap);
  va_end(ap);
}
int hb_alloc_state(sb200_graph* g);
int hb_reset(sb200_graph* g);
int hb_set_l2_window(sb200_graph* g, uint64_t want);
int hb_step(sb200_graph* g, sb200_iter_stats* st);
int hb_step_launch(sb200_graph* g, bool with_barrier);
int hb_step_finish(sb200_graph* g, sb200_iter_stats* st);
int hb_barrier(sb200_graph* g);
__global__ void k_owned_flags(const uint32_t* __restrict__ inv, const uint32_t* __restrict__ sub, uint64_t N, uint32_t world, uint32_t rank,
                              uint8_t* owned, uint32_t* sub_out) {
  const uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;   // r = position in ascending-id order
  if (r >= N) return;
  const uint32_t v = inv[r];
  if (owned) owned[r] = (world <= 1 || ((v >> 5) % world) == rank) ? 1 : 0;
  if (sub_out) sub_out[r] = sub ? sub[v] : (world <= 1 ? 1u : 0xFFFFFFFFu >> (32 - world));
}
int hb_result(sb200_graph* g, uint64_t* id_lo, uint64_t* id_hi, double* cent, uint64_t cap, uint64_t* len);
int hb_registers(sb200_graph* g, uint64_t first, uint64_t count, uint8_t* out);
int hb_ranked(sb200_graph* g, int ties_desc, uint64_t* id_lo, uint64_t* id_hi, double* cent, uint64_t cap, uint64_t* len);
int hb_kahan(sb200_graph* g, uint64_t first, uint64_t count, double* sum, double* err);
}  // namespace sb200
using namespace sb200;

uint64_t sb200_graph::hbm_bytes() const {
  return id_lo.bytes() + id_hi.bytes() + perm.bytes() + inv.bytes() + row_ptr.bytes() + col.bytes() + fwd_ptr.bytes() +
         fwd_dst.bytes() + item_row.bytes() + item_start.bytes() + partial.bytes() + regs[0].bytes() + regs[1].bytes() +
         seed.bytes() + bm[0].bytes() + bm[1].bytes() + size_cache.bytes() + kahan_sum.bytes() + kahan_err.bytes() +
         frontier_list.bytes() + frontier_off.bytes() + frontier_scan.bytes() + cub_tmp.bytes() + counters.bytes() + sub_mask.bytes() + sync_page.bytes();
}

extern "C" {

const char* sb200_last_error(void) { return t_err; }
#ifndef SB200_EMU
const char* sb200_version(void) { return "stract_b200 0.1 (sm_90a)"; }
#else
const char* sb200_version(void) { return "stract_b200 0.1 CPU SIMT emulation (tests/emu, tests only)"; }
#endif
uint64_t sb200_kernel_launch_count(void) { return g_launches.load(); }

#define SB_ENTER(g)                                            \
  if (!(g)) SB_FAIL(SB200_EINVAL, "NULL graph handle");        \
  SB_CUDA(cudaSetDevice((g)->device))

int sb200_graph_create(const uint64_t* from_lo, const uint64_t* from_hi, const uint64_t* to_lo, const uint64_t* to_hi,
                       const uint64_t* rel_flags, uint64_t n_edges, uint64_t skipped_rel_mask, int device, int rank,
                       int world_size, sb200_graph** out) {
  if (!out) SB_FAIL(SB200_EINVAL, "out is NULL");
  *out = nullptr;
  if (world_size < 1 || world_size > 64 || rank < 0 || rank >= world_size)
    SB_FAIL(SB200_EINVAL, "bad rank/world_size %d/%d", rank, world_size);
  int ndev = 0;
  SB_CUDA(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) SB_FAIL(SB200_EINVAL, "device %d not in [0,%d)", device, ndev);
  SB_CUDA(cudaSetDevice(device));
  sb200_graph* g = new (std::nothrow) sb200_graph();
  if (!g) SB_FAIL(SB200_ENOMEM, "host allocation failed");
  g->device = device; g->rank = rank; g->world = world_size;
  int rc = SB200_OK;
  auto body = [&]() -> int {
    SB_CUDA(cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking));
    SB_CUDA(cudaEventCreate(&g->ev0)); SB_CUDA(cudaEventCreate(&g->ev1));
    SB_CUDA(cudaEventCreate(&g->ev_run0)); SB_CUDA(cudaEventCreate(&g->ev_run1));
    for (int f = 0; f < sb200_graph::F_COUNT; f++) { SB_CUDA(cudaEventCreate(&g->prof_ev[f][0])); SB_CUDA(cudaEventCreate(&g->prof_ev[f][1])); }
    {
      // staging temporaries and the CSR come from the stream-ordered pool (kept warm across creates);
      // the register arrays / bitmaps below stay plain cudaMalloc because they are exported through CUDA IPC
      static bool pool_ready[64] = {false};
      if (device < 64 && !pool_ready[device]) {
        cudaMemPool_t pool; uint64_t keep = ~0ull;
        SB_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
        SB_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
        pool_ready[device] = true;
      }
      PoolScope scope(getenv("SB200_NO_POOL") ? nullptr : g->stream);
      SB_TRY(stage_graph(g, from_lo, from_hi, to_lo, to_hi, rel_flags, n_edges, skipped_rel_mask));
    }
    g->cub_tmp.release();
    {
      // a single-rank handle never exports its arrays, so they can come from the warm pool too (saves the
      // cudaMalloc/cudaFree of ~4.5 GB per create/destroy at C2 size); sharded handles need IPC-exportable memory
      PoolScope scope((world_size == 1 && !getenv("SB200_NO_POOL")) ? g->stream : nullptr);
      SB_TRY(hb_alloc_state(g));
    }
    SB_TRY(hb_reset(g));
    return SB200_OK;
  };
  rc = body();
  if (rc != SB200_OK) { sb200_graph_destroy(g); return rc; }
  *out = g;
  return SB200_OK;
}

void sb200_graph_destroy(sb200_graph* g) {
  if (!g) return;
  cudaSetDevice(g->device);
  if (g->stream) cudaStreamSynchronize(g->stream);
  if (g->peers_ipc) for (int p = 0; p < g->n_peers; p++) for (int i = 0; i < 2; i++) {
    if (g->peer_regs[i][p]) cudaIpcCloseMemHandle(g->peer_regs[i][p]);
    if (g->peer_bm[i][p]) cudaIpcCloseMemHandle(g->peer_bm[i][p]);
  }
  if (g->peers_ipc) for (int p = 0; p < g->n_peers; p++) if (g->peer_sync[p]) cudaIpcCloseMemHandle(g->peer_sync[p]);
  if (g->l2_window_bytes) cudaCtxResetPersistingL2Cache();  // hand the pinned hub lines back to the normal L2
  if (g->h_counters) cudaFreeHost(g->h_counters);
  if (g->ev0) cudaEventDestroy(g->ev0);
  if (g->ev1) cudaEventDestroy(g->ev1);
  if (g->side_stream) { cudaStreamSynchronize(g->side_stream); cudaStreamDestroy(g->side_stream); }
  if (g->ev_fork) cudaEventDestroy(g->ev_fork);
  if (g->ev_join) cudaEventDestroy(g->ev_join);
  for (int k = 0; k < 2; k++) if (g->side_prof[k]) cudaEventDestroy(g->side_prof[k]);
  if (g->ev_run0) cudaEventDestroy(g->ev_run0);
  if (g->ev_run1) cudaEventDestroy(g->ev_run1);
  for (int f = 0; f < sb200_graph::F_COUNT; f++) for (int k = 0; k < 2; k++) if (g->prof_ev[f][k]) cudaEventDestroy(g->prof_ev[f][k]);
  cudaStream_t s = g->stream;
  const int dev = g->device;
  delete g;  // DevBuf destructors free HBM
  if (s) { arena_retire_stream(dev, s); cudaStreamDestroy(s); }  // the stream is idle: its arena blocks are free for all
}

int sb200_graph_get_info(const sb200_graph* g, sb200_graph_info* info) {
  if (!g || !info) SB_FAIL(SB200_EINVAL, "NULL argument");
  info->n_nodes = g->N; info->n_edges_input = g->E_in; info->n_edges_kept = g->E_kept; info->n_edges_local = g->E_local;
  info->row_begin = 0; info->row_end = g->N; info->hbm_bytes = g->hbm_bytes(); info->stage_ms = g->stage_ms;
  return SB200_OK;
}

int sb200_hyperball_set_policy(sb200_graph* g, double dense_frac, double push_div, int force_mode) {
  if (!g) SB_FAIL(SB200_EINVAL, "NULL graph handle");
  if (dense_frac >= 0) g->dense_frac = dense_frac;
  if (push_div > 0) g->push_div = push_div;
  g->force_mode = force_mode;
  return SB200_OK;
}

int sb200_hyperball_set_option(sb200_graph* g, const char* name, double value) {
  if (!g || !name) SB_FAIL(SB200_EINVAL, "NULL graph handle or option name");
  if (g->step_in_flight) SB_FAIL(SB200_ESTATE, "an iteration is in flight");
  if (!strcmp(name, "quad_side_ctas")) { if (value < 0 || value > 16) SB_FAIL(SB200_EINVAL, "quad_side_ctas must be 0..16"); g->opt_side_ctas = (int)value; }
  else if (!strcmp(name, "owned_items")) g->opt_owned_list = value != 0.0 ? 1 : 0;
  else if (!strcmp(name, "publish_all")) g->publish_all = value != 0.0;
  else if (!strcmp(name, "l2_window_mb")) {
    if (!(value >= 0 && value <= 1024)) SB_FAIL(SB200_EINVAL, "l2_window_mb must be 0..1024");
    SB_CUDA(cudaSetDevice(g->device));   // the persisting set-aside is a setting of the handle's device
    SB_TRY(sb200::hb_set_l2_window(g, (uint64_t)(value * (1 << 20))));
  }
  else if (!strcmp(name, "l1_hub_kb")) {
    // 0: every gather bypasses L1; at least N * 64 / 1024: every gather goes through L1
    if (!(value >= 0 && value <= 1073741824.0)) SB_FAIL(SB200_EINVAL, "l1_hub_kb must be 0..1073741824");
    g->l1_hub_bytes = (uint64_t)(value * 1024);
  }
  else SB_FAIL(SB200_EINVAL, "unknown option '%s'", name);
  return SB200_OK;
}

int sb200_hyperball_reset(sb200_graph* g) { SB_ENTER(g); g->reuse++; return hb_reset(g); }

int sb200_hyperball_step(sb200_graph* g, sb200_iter_stats* stats) { SB_ENTER(g); return hb_step(g, stats); }

int sb200_hyperball_run(sb200_graph* g, uint32_t max_iters, uint32_t* iters_done, sb200_iter_stats* per_iter, uint32_t cap) {
  SB_ENTER(g);
  if (g->world != 1) SB_FAIL(SB200_ESTATE, "sb200_hyperball_run drives single-rank handles; sharded handles step + exchange");
  uint32_t n = 0;
  SB_CUDA(cudaEventRecord(g->ev_run0, g->stream));
  // calculate_centrality loop, harmonic.rs:237-280: stop after the first iteration without changes
  while (g->has_changes && (max_iters == 0 || g->t < max_iters)) {
    // registers only grow and are bounded, so the loop always ends; the cap only guards against a broken build
    if (g->t >= 100000) SB_FAIL(SB200_ESTATE, "HyperBall did not converge within 100000 iterations");
    sb200_iter_stats st;
    SB_TRY(hb_step(g, &st));
    if (per_iter && n < cap) per_iter[n] = st;
    n++;
  }
  SB_CUDA(cudaEventRecord(g->ev_run1, g->stream));
  SB_CUDA(cudaStreamSynchronize(g->stream));
  cudaEventElapsedTime(&g->last_run_ms, g->ev_run0, g->ev_run1);
  if (iters_done) *iters_done = g->t;
  return SB200_OK;
}

int sb200_hyperball_last_run_ms(sb200_graph* g, float* ms) {
  if (!g || !ms) SB_FAIL(SB200_EINVAL, "NULL argument");
  *ms = g->last_run_ms;
  return SB200_OK;
}

int sb200_hyperball_set_profiling(sb200_graph* g, int on) {
  if (!g) SB_FAIL(SB200_EINVAL, "NULL graph handle");
  g->profiling = on != 0;
  for (int f = 0; f < sb200_graph::F_COUNT; f++) { g->prof_launches[f] = 0; g->prof_ms[f] = 0; g->prof_bytes[f] = 0; g->prof_used[f] = false; }
  return SB200_OK;
}

int sb200_hyperball_get_profile(sb200_graph* g, sb200_kernel_prof* out, uint32_t cap, uint32_t* n) {
  if (!g || !n) SB_FAIL(SB200_EINVAL, "NULL argument");
  static const char* names[sb200_graph::F_COUNT] = {"k_pull_warp<dense>", "k_pull_quad<dense>", "k_pull_warp<frontier>",
                                                     "k_pull_quad<frontier>", "k_pull_merge", "k_push", "k_finalize",
                                                     "k_pull_warp<seed>", "k_pull_quad<seed>"};
  uint32_t k = 0;
  for (int f = 0; f < sb200_graph::F_COUNT; f++) {
    if (out && k < cap) {
      memset(&out[k], 0, sizeof(out[k]));
      strncpy(out[k].name, names[f], sizeof(out[k].name) - 1);
      out[k].launches = g->prof_launches[f]; out[k].ms = g->prof_ms[f]; out[k].alg_bytes = g->prof_bytes[f];
    }
    k++;
  }
  *n = k;
  return SB200_OK;
}

int sb200_hyperball_result(sb200_graph* g, uint64_t* id_lo, uint64_t* id_hi, double* centrality, uint64_t cap, uint64_t* len) {
  SB_ENTER(g);
  if (!len) SB_FAIL(SB200_EINVAL, "len is NULL");
  if (centrality && (!id_lo || !id_hi)) SB_FAIL(SB200_EINVAL, "id outputs are NULL");
  return hb_result(g, id_lo, id_hi, centrality, cap, len);
}

int sb200_hyperball_ranked(sb200_graph* g, int ties_desc, uint64_t* id_lo, uint64_t* id_hi, double* centrality, uint64_t cap, uint64_t* len) {
  SB_ENTER(g);
  if (!len) SB_FAIL(SB200_EINVAL, "len is NULL");
  if (centrality && (!id_lo || !id_hi)) SB_FAIL(SB200_EINVAL, "id outputs are NULL");
  return hb_ranked(g, ties_desc, id_lo, id_hi, centrality, cap, len);
}

int sb200_hyperball_registers(sb200_graph* g, uint64_t first, uint64_t count, uint8_t* out) { SB_ENTER(g); return hb_registers(g, first, count, out); }
int sb200_hyperball_kahan(sb200_graph* g, uint64_t first, uint64_t count, double* sum, double* err) { SB_ENTER(g); return hb_kahan(g, first, count, sum, err); }

int sb200_graph_node_ids(sb200_graph* g, uint64_t first, uint64_t count, uint64_t* id_lo, uint64_t* id_hi) {
  SB_ENTER(g);
  if (first + count > g->N) SB_FAIL(SB200_EINVAL, "range outside the node set");
  if (!count) return SB200_OK;
  SB_CUDA(cudaMemcpyAsync(id_lo, g->id_lo.p + first, count * 8, cudaMemcpyDefault, g->stream));
  SB_CUDA(cudaMemcpyAsync(id_hi, g->id_hi.p + first, count * 8, cudaMemcpyDefault, g->stream));
  SB_CUDA(cudaStreamSynchronize(g->stream));
  return SB200_OK;
}

int sb200_hyperball_exchange_ptrs(sb200_graph* g, void** regs, uint64_t* regs_bytes, void** frontier_words, uint64_t* frontier_bytes) {
  SB_ENTER(g);
  if (regs) *regs = g->regs[g->cur].p;
  if (regs_bytes) *regs_bytes = g->N * 64;
  if (frontier_words) *frontier_words = g->bm[g->bcur].p;
  if (frontier_bytes) *frontier_bytes = ((g->N + 31) / 32) * 4;
  return SB200_OK;
}
int sb200_graph_row_ranges(sb200_graph* g, uint64_t* begins) {
  if (!g || !begins) SB_FAIL(SB200_EINVAL, "NULL argument");
  for (int r = 0; r <= g->world; r++) begins[r] = r == g->world ? g->N : 0;
  return SB200_OK;
}
// ---- fused exchange over NVLink peer memory (CUDA IPC between the per-GPU processes) ----------------------
int sb200_hyperball_ipc_export(sb200_graph* g, uint8_t* out /* SB200_IPC_BLOB_BYTES */) {
  SB_ENTER(g);
  if (!out) SB_FAIL(SB200_EINVAL, "out is NULL");
  if (g->world < 2 || !g->sync_page.p) SB_FAIL(SB200_ESTATE, "only sharded handles (world_size > 1) export their state");
  memset(out, 0, SB200_IPC_BLOB_BYTES);
  void* ptrs[5] = {g->regs[0].p, g->regs[1].p, g->bm[0].p, g->bm[1].p, g->sync_page.p};
  for (int i = 0; i < 5; i++) {
    cudaIpcMemHandle_t h;
    SB_CUDA(cudaIpcGetMemHandle(&h, ptrs[i]));
    static_assert(sizeof(h) == SB200_IPC_HANDLE_BYTES, "IPC handle size");
    memcpy(out + (size_t)i * SB200_IPC_HANDLE_BYTES, &h, sizeof(h));
  }
  const uint32_t tail[2] = {(uint32_t)g->rank, (uint32_t)g->world};
  memcpy(out + 5 * SB200_IPC_HANDLE_BYTES, tail, sizeof(tail));
  return SB200_OK;
}
int sb200_hyperball_ipc_import(sb200_graph* g, const uint8_t* blob) {
  SB_ENTER(g);
  if (!blob) SB_FAIL(SB200_EINVAL, "blob is NULL");
  if (!g->peers_ipc) SB_FAIL(SB200_ESTATE, "publish targets were set by address; IPC import cannot be mixed in");
  if (g->n_peers >= sb200::MAX_PEERS) SB_FAIL(SB200_ERANGE, "more than %d peers", sb200::MAX_PEERS);
  uint32_t tail[2];
  memcpy(tail, blob + 5 * SB200_IPC_HANDLE_BYTES, sizeof(tail));
  if ((int)tail[1] != g->world || (int)tail[0] >= g->world || (int)tail[0] == g->rank)
    SB_FAIL(SB200_EINVAL, "blob of rank %u / world %u does not fit this handle (rank %d / world %d)", tail[0], tail[1], g->rank, g->world);
  for (int p = 0; p < g->n_peers; p++) if (g->peer_rank[p] == (int)tail[0]) SB_FAIL(SB200_ESTATE, "rank %u imported twice", tail[0]);
  void* opened[5];
  for (int i = 0; i < 5; i++) {
    cudaIpcMemHandle_t h;
    memcpy(&h, blob + (size_t)i * SB200_IPC_HANDLE_BYTES, sizeof(h));
    SB_CUDA(cudaIpcOpenMemHandle(&opened[i], h, cudaIpcMemLazyEnablePeerAccess));
  }
  const int p = g->n_peers++;
  g->peer_regs[0][p] = opened[0]; g->peer_regs[1][p] = opened[1];
  g->peer_bm[0][p] = opened[2]; g->peer_bm[1][p] = opened[3];
  g->peer_sync[p] = opened[4];
  g->peer_rank[p] = (int)tail[0];
  return SB200_OK;
}
int sb200_hyperball_p2p_enable(sb200_graph* g, int on) {
  SB_ENTER(g);
  if (on && g->n_peers != g->world - 1) SB_FAIL(SB200_ESTATE, "imported %d peers, world_size-1 = %d", g->n_peers, g->world - 1);
  g->p2p = on != 0;
  return SB200_OK;
}

// ---- caller-owned state + publish targets by address (symmetric / multicast memory) -----------------------
int sb200_hyperball_state_bytes(sb200_graph* g, uint64_t* regs_bytes, uint64_t* bitmap_bytes) {
  if (!g) SB_FAIL(SB200_EINVAL, "NULL graph handle");
  if (regs_bytes) *regs_bytes = std::max<uint64_t>(g->N, 1) * 64;
  if (bitmap_bytes) *bitmap_bytes = ((g->N + 31) / 32 + 1) * 4;
  return SB200_OK;
}
int sb200_hyperball_bind_state(sb200_graph* g, void* regs0, void* regs1, void* bitmap0, void* bitmap1) {
  SB_ENTER(g);
  if (!regs0 || !regs1 || !bitmap0 || !bitmap1) SB_FAIL(SB200_EINVAL, "NULL state buffer");
  if (regs0 == regs1 || bitmap0 == bitmap1) SB_FAIL(SB200_EINVAL, "the two register arrays / bitmaps must be distinct");
  if (((uintptr_t)regs0 | (uintptr_t)regs1) & 63) SB_FAIL(SB200_EINVAL, "register arrays must be 64-byte aligned");
  if (((uintptr_t)bitmap0 | (uintptr_t)bitmap1) & 3) SB_FAIL(SB200_EINVAL, "bitmaps must be 4-byte aligned");
  void* all[4] = {regs0, regs1, bitmap0, bitmap1};
  for (void* q : all) if (!is_device_ptr(q)) SB_FAIL(SB200_EINVAL, "state buffers must be device memory");
  if (g->t != 0 || g->exchange_pending) SB_FAIL(SB200_ESTATE, "bind the state right after create/reset, before the first step");
  if (g->n_peers) SB_FAIL(SB200_ESTATE, "bind the state before the publish targets are set");
  SB_CUDA(cudaStreamSynchronize(g->stream));
  const uint64_t rn = std::max<uint64_t>(g->N, 1) * 64, bn = (g->N + 31) / 32 + 1;
  g->regs[0].adopt((uint8_t*)regs0, rn); g->regs[1].adopt((uint8_t*)regs1, rn);
  g->bm[0].adopt((uint32_t*)bitmap0, bn); g->bm[1].adopt((uint32_t*)bitmap1, bn);
  return hb_reset(g);
}
int sb200_hyperball_set_publish_targets(sb200_graph* g, int n_targets, const uint64_t* regs0, const uint64_t* regs1,
                                        const uint64_t* bitmap0, const uint64_t* bitmap1) {
  SB_ENTER(g);
  if (n_targets < 0 || n_targets > sb200::MAX_PEERS) SB_FAIL(SB200_ERANGE, "n_targets %d not in [0,%d]", n_targets, sb200::MAX_PEERS);
  if (n_targets && (!regs0 || !regs1 || !bitmap0 || !bitmap1)) SB_FAIL(SB200_EINVAL, "NULL target array");
  if (g->n_peers && g->peers_ipc) SB_FAIL(SB200_ESTATE, "IPC peers were imported; targets by address cannot be mixed in");
  if (g->exchange_pending) SB_FAIL(SB200_ESTATE, "an exchange is pending");
  for (int p = 0; p < n_targets; p++) {
    if (!regs0[p] || !regs1[p] || !bitmap0[p] || !bitmap1[p]) SB_FAIL(SB200_EINVAL, "target %d has a NULL address", p);
    if ((regs0[p] | regs1[p]) & 15) SB_FAIL(SB200_EINVAL, "target %d: register arrays must be 16-byte aligned", p);
  }
  for (int p = 0; p < sb200::MAX_PEERS; p++) {
    const bool on = p < n_targets;
    g->peer_regs[0][p] = on ? (void*)(uintptr_t)regs0[p] : nullptr; g->peer_regs[1][p] = on ? (void*)(uintptr_t)regs1[p] : nullptr;
    g->peer_bm[0][p] = on ? (void*)(uintptr_t)bitmap0[p] : nullptr; g->peer_bm[1][p] = on ? (void*)(uintptr_t)bitmap1[p] : nullptr;
  }
  g->n_peers = n_targets; g->peers_ipc = false; g->p2p = n_targets > 0;
  // world_size-1 unicast targets are taken in rank order (own rank left out); any other count (e.g. the single
  // multicast mapping) reaches every replica at once, so the subscriber filter is off
  if (n_targets == g->world - 1) { for (int p = 0; p < n_targets; p++) g->peer_rank[p] = p < g->rank ? p : p + 1; g->publish_all = false; }
  else g->publish_all = true;
  return SB200_OK;
}

// ---- the round loop behind the ABI ---------------------------------------------------------------------------
// (a) one process, n handles (n GPUs of one box, or -- for tests -- several ranks on one GPU): link wires every
//     handle's publish targets to the other handles' arrays by address, run drives the rounds.
int sb200_hyperball_group_link(sb200_graph** hs, int n) {
  if (!hs || n < 1) SB_FAIL(SB200_EINVAL, "bad group");
  for (int i = 0; i < n; i++) {
    if (!hs[i]) SB_FAIL(SB200_EINVAL, "NULL handle %d", i);
    if (hs[i]->world != n || hs[i]->rank != i) SB_FAIL(SB200_EINVAL, "handle %d has rank %d / world %d; expected rank %d / world %d", i, hs[i]->rank, hs[i]->world, i, n);
    if (hs[i]->N != hs[0]->N || hs[i]->E_kept != hs[0]->E_kept) SB_FAIL(SB200_EINVAL, "handle %d was staged from a different graph", i);
    if (hs[i]->n_peers) SB_FAIL(SB200_ESTATE, "handle %d already has publish targets", i);
  }
  if (n == 1) return SB200_OK;
  if (n - 1 > sb200::MAX_PEERS) SB_FAIL(SB200_ERANGE, "more than %d peers", sb200::MAX_PEERS);
  for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) {
    if (i == j || hs[i]->device == hs[j]->device) continue;
    int can = 0;
    SB_CUDA(cudaDeviceCanAccessPeer(&can, hs[i]->device, hs[j]->device));
    if (!can) SB_FAIL(SB200_ESTATE, "device %d cannot access device %d", hs[i]->device, hs[j]->device);
    SB_CUDA(cudaSetDevice(hs[i]->device));
    const cudaError_t e = cudaDeviceEnablePeerAccess(hs[j]->device, 0);
    if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) SB_CUDA(e);
    cudaGetLastError();
  }
  for (int i = 0; i < n; i++) {
    sb200_graph* g = hs[i];
    int p = 0;
    for (int j = 0; j < n; j++) {
      if (j == i) continue;
      g->peer_regs[0][p] = hs[j]->regs[0].p; g->peer_regs[1][p] = hs[j]->regs[1].p;
      g->peer_bm[0][p] = hs[j]->bm[0].p; g->peer_bm[1][p] = hs[j]->bm[1].p;
      g->peer_sync[p] = hs[j]->sync_page.p; g->peer_rank[p] = j;
      p++;
    }
    g->n_peers = n - 1; g->peers_ipc = false; g->p2p = true;
  }
  return SB200_OK;
}

int sb200_hyperball_group_run(sb200_graph** hs, int n, uint32_t max_iters, uint32_t* iters_done, sb200_iter_stats* per_iter, uint32_t cap) {
  if (!hs || n < 1) SB_FAIL(SB200_EINVAL, "bad group");
  for (int i = 0; i < n; i++) if (!hs[i] || hs[i]->world != n || hs[i]->rank != i) SB_FAIL(SB200_EINVAL, "handle %d does not belong to a group of %d", i, n);
  for (int i = 0; i < n; i++) if (n > 1 && (!hs[i]->p2p || hs[i]->n_peers != n - 1)) SB_FAIL(SB200_ESTATE, "call sb200_hyperball_group_link first");
  for (int i = 0; i < n; i++) { SB_CUDA(cudaSetDevice(hs[i]->device)); SB_CUDA(cudaStreamSynchronize(hs[i]->stream)); }  // every replica initialised
  uint32_t t = 0;
  bool changes = hs[0]->N > 0 && hs[0]->has_changes;
  // coordinator.rs:151-213: rounds until one leaves Meta.round_had_changes unset
  while (changes && (max_iters == 0 || t < max_iters)) {
    if (t >= 100000) SB_FAIL(SB200_ESTATE, "HyperBall did not converge within 100000 iterations");
    for (int i = 0; i < n; i++) { SB_CUDA(cudaSetDevice(hs[i]->device)); SB_TRY(hb_step_launch(hs[i], false)); }
    uint64_t total = 0;
    for (int i = 0; i < n; i++) {
      sb200_iter_stats st;
      SB_CUDA(cudaSetDevice(hs[i]->device));
      SB_TRY(hb_step_finish(hs[i], &st));
      total += st.n_changed;
      if (per_iter && t < cap) per_iter[(size_t)i * cap + t] = st;
    }
    for (int i = 0; i < n; i++) { hs[i]->n_changed_prev = total; hs[i]->has_changes = total != 0; hs[i]->exchange_pending = false; }
    changes = total != 0;
    t++;
  }
  if (iters_done) *iters_done = t;
  return SB200_OK;
}

// (b) one process per GPU: every rank calls this at the same time after the IPC blobs have been exchanged and
//     sb200_hyperball_p2p_enable.  No host-side collective is involved: the ranks meet in k_barrier_count.
int sb200_hyperball_run_sharded(sb200_graph* g, uint32_t max_iters, uint32_t* iters_done, sb200_iter_stats* per_iter, uint32_t cap) {
  SB_ENTER(g);
  if (g->world < 2) return sb200_hyperball_run(g, max_iters, iters_done, per_iter, cap);
  if (!g->p2p || g->n_peers != g->world - 1) SB_FAIL(SB200_ESTATE, "exchange the IPC blobs of all %d peers and enable p2p first", g->world - 1);
  SB_CUDA(cudaEventRecord(g->ev_run0, g->stream));
  SB_TRY(hb_barrier(g));
  uint32_t n = 0;
  while (g->has_changes && (max_iters == 0 || g->t < max_iters)) {
    if (g->t >= 100000) SB_FAIL(SB200_ESTATE, "HyperBall did not converge within 100000 iterations");
    sb200_iter_stats st;
    SB_TRY(hb_step_launch(g, true));
    SB_TRY(hb_step_finish(g, &st));
    if (per_iter && n < cap) per_iter[n] = st;
    n++;
  }
  SB_CUDA(cudaEventRecord(g->ev_run1, g->stream));
  SB_CUDA(cudaStreamSynchronize(g->stream));
  cudaEventElapsedTime(&g->last_run_ms, g->ev_run0, g->ev_run1);
  if (iters_done) *iters_done = g->t;
  return SB200_OK;
}

// which nodes this rank owns / which ranks read each node's row, in ascending-id order (parity checks of sharded handles)
int sb200_graph_ownership(sb200_graph* g, uint8_t* owned /* nullable, n_nodes */, uint32_t* subscribers /* nullable, n_nodes */) {
  SB_ENTER(g);
  const uint64_t N = g->N;
  if (!N) return SB200_OK;
  DevBuf<uint8_t> o; DevBuf<uint32_t> m;
  if (owned) SB_TRY(o.alloc(N));
  if (subscribers) SB_TRY(m.alloc(N));
  SB_LAUNCH(k_owned_flags, div_up(N, 256), 256, 0, g->stream, g->inv.p, (g->publish_all || !g->sub_mask.p) ? (const uint32_t*)nullptr : g->sub_mask.p, N,
            (uint32_t)g->world, (uint32_t)g->rank, owned ? o.p : (uint8_t*)nullptr, subscribers ? m.p : (uint32_t*)nullptr);
  SB_CHECK_LAUNCH();
  if (owned) SB_CUDA(cudaMemcpyAsync(owned, o.p, N, cudaMemcpyDefault, g->stream));
  if (subscribers) SB_CUDA(cudaMemcpyAsync(subscribers, m.p, N * 4, cudaMemcpyDefault, g->stream));
  SB_CUDA(cudaStreamSynchronize(g->stream));
  return SB200_OK;
}

int sb200_hyperball_exchange_done(sb200_graph* g, uint64_t global_n_changed) {
  SB_ENTER(g);
  g->n_changed_prev = global_n_changed;
  g->has_changes = global_n_changed != 0;
  g->exchange_pending = false;
  return SB200_OK;
}

}  // extern "C"
