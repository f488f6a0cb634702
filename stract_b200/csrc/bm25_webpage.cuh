// bm25_webpage.cuh -- the recall webpages of Stract's searcher (sb200_multi_signal_webpages): for a GIVEN list of documents
// per query, what LocalRecallRankingWebpage::new (core/src/ranking/pipeline/stages/recall.rs:167-220) takes from the
// SignalComputer -- every signal's (value, score) (compute_signals), the optic boost (boosts, computer/mod.rs:471-497) -- and what
// TitleDistanceScorer / BodyDistanceScorer (pipeline/scorers/term_distance.rs) make of get_field_positions: the min slop of the
// Title and CleanBody query terms.
//
// The documents of every query are sorted ascending (CUB radix sort of (query << 32 | doc) keys carrying the caller's index),
// because a posting cursor only moves forward; every output goes back through that index, so outputs follow the caller's order.
//   k_wp_signals  one warp per 32 consecutive sorted documents of one query: seeks every slot to them (pl_seek_at, the cursor of
//                 k_plan_recall) and, for the text slots of the two distance fields, records each posting's position offset (its
//                 block's base from the positions directory plus the tfs before it in the block, as k_phrase_cand does).  Then
//                 every lane runs m_total (bm25_multi.cuh) on its document with a sink that keeps each op's value / score and the
//                 boost factor.  A (document, distance field) with >= 2 slots that all hold the document goes to the work list;
//                 every other one is decided as u32::MAX on the spot.
//   k_wp_slop     one warp per work item: decodes each slot's positions (ph_read_deltas + ph_prefix from 0: positions_with_offset(0))
//                 into shared memory -- a list set that does not fit goes to a second pass over global scratch -- then per
//                 consecutive slot pair every lane takes positions a of the left list and binary-searches the smallest b > a in
//                 the right one; a warp min of b - a is the pair's slop and the result the max over the pairs.  This equals
//                 min_slop_two_positions' two-cursor walk (DESIGN.md §3): whenever the walk records b - a, its b cursor is the
//                 smallest b > a (it only passes values <= an earlier a <= a), and it stops once no later b exists.
#pragma once

namespace sb200 {

template <int TMAX>
__host__ __device__ constexpr size_t wp_warp_smem() { return pl_warp_smem<TMAX>() + (size_t)TMAX * 128 * 4; }
template <int TMAX>
__host__ __device__ constexpr size_t wp_cta_smem() { return M_MAX_FIELDS * 256 * 4 + M_MAX_OPS * sizeof(MOp) + WQ * wp_warp_smem<TMAX>(); }

struct WpParams {
  MParams M;                                // fields, ops, slots per query (text slots first), optic rule tables by query
  const uint64_t* keys; const uint32_t* idx;   // sorted (q << 32 | doc) and the caller's flat index q * n_docs_max + i
  const uint32_t* q_beg;                    // [n_queries + 1] each query's range of keys
  const uint32_t* units; uint32_t n_units;  // first key of every chunk of <= 32 keys of one query
  uint32_t dist[2];                         // field index of Title / CleanBody, SB200_WEBPAGE_NO_FIELD when not registered
  const uint64_t* pos_base[2];              // per posting block slot of the distance field: position offset of its first posting
  uint32_t nd;                              // row width of the offset scratch: distance slots per query, at most
  uint64_t* s_off; uint32_t* s_tf;          // [key][nd]
  double* o_values; double* o_scores; double* o_boosts; uint32_t* o_slop;   // by caller index
  unsigned long long* work;                 // (key << 1 | field) of the pairs that need positions
  unsigned long long* counters;             // [0] work items [1] format errors [2] documents with a work item
};

// the position-offset observer of pl_seek_at: `base` NULL for slots outside the distance fields
struct WpPos {
  uint32_t* pre; const uint64_t* base; uint32_t first; uint64_t off;
  __device__ __forceinline__ void block(const uint32_t* tfs, uint32_t lane) {
    if (!base) return;   // warp-uniform
    const uint4 f = ((const uint4*)tfs)[lane];
    const uint32_t loc = f.x + f.y + f.z + f.w;
    const uint32_t ex = warp_scan_incl(loc, lane) - loc;
    ((uint4*)pre)[lane] = make_uint4(ex, ex + f.x, ex + f.x + f.y, ex + f.x + f.y + f.z);
    __syncwarp();
  }
  __device__ __forceinline__ void hit(uint32_t j, uint32_t jj) { if (base) off = base[first + j] + pre[jj]; }
};

__device__ uint64_t wp_seek(const PSeg& G, const OTerm& c, uint32_t* cur_p, uint32_t* cached_p, uint32_t* docs, uint32_t* tfs, uint32_t* bloom,
                            uint32_t d, bool want, uint32_t lane, WpPos& pos) {
  return pl_seek_at(G, c, cur_p, cached_p, docs, tfs, bloom, d, want, lane, pos);
}

// m_total's sink: the ops' value / score straight into the caller-ordered outputs, the boost factors multiplied up
struct WpSink {
  static constexpr bool ACTIVE = true;
  double* v; double* s; double b;
  __device__ __forceinline__ void op(const MOp& op, uint32_t o, double value, double score) {
    if (op.kind != 4u) v[o] = value;   // a numeric CoreSignal's value is its raw column, which the caller holds
    s[o] = score;
  }
  __device__ __forceinline__ void boost(double f) { b = __dmul_rn(b, f); }
};

template <int TMAX>
__global__ void __launch_bounds__(WQ * 32) k_wp_signals(const WpParams W) {
  const MParams& P = W.M;
  SB_DYN_SMEM(smem_raw);
  float* s_cache = (float*)smem_raw;                                   // [M_MAX_FIELDS][256]
  MOp* s_ops = (MOp*)(smem_raw + M_MAX_FIELDS * 256 * 4);              // [M_MAX_OPS]
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char* wbase = smem_raw + M_MAX_FIELDS * 256 * 4 + M_MAX_OPS * sizeof(MOp) + warp * wp_warp_smem<TMAX>();
  uint32_t* docs = (uint32_t*)wbase;                                   // [TMAX][128]
  uint32_t* tfs = docs + TMAX * 128;                                   // [TMAX][128]
  uint32_t* pre = tfs + TMAX * 128;                                    // [TMAX][128] tfs before each entry (distance slots)
  uint32_t* bloom = pre + TMAX * 128;                                  // [TMAX][16]
  OTerm* tc = (OTerm*)(bloom + TMAX * 16);                             // [TMAX]
  float* s_wf = (float*)(tc + TMAX);                                   // [TMAX]
  uint32_t* s_fld = (uint32_t*)(s_wf + TMAX);                          // [TMAX]
  uint32_t* s_cur = s_fld + TMAX;                                      // [TMAX]
  uint32_t* s_cached = s_cur + TMAX;                                   // [TMAX]
  uint32_t* s_nf = s_cached + TMAX;                                    // [M_MAX_FIELDS]
  for (uint32_t i = threadIdx.x; i < P.n_fields * 256; i += WQ * 32) s_cache[i] = P.fields[i >> 8].cache[i & 255];
  for (uint32_t i = threadIdx.x; i < P.n_ops; i += WQ * 32) s_ops[i] = P.ops[i];
  __syncthreads();  // the only block barrier
  const uint32_t u = blockIdx.x * WQ + warp;
  if (u >= W.n_units) return;
  const uint32_t first = W.units[u];
  const uint32_t q = (uint32_t)(W.keys[first] >> 32);
  const uint32_t end = min(W.q_beg[q + 1], first + 32u);
  const uint32_t e = first + lane;
  const bool live = e < end;
  const uint32_t d = live ? (uint32_t)W.keys[e] : 0xFFFFFFFFu;
  const uint32_t at = live ? W.idx[e] : 0u;
  const uint32_t SM = P.n_slots_max;
  const uint32_t T = min(P.q_nslots[q], (uint32_t)TMAX);
  const uint32_t o_nr = P.d_nrules ? P.d_nrules[q] : 0u;
  if (lane < M_MAX_FIELDS) s_nf[lane] = 0;
  __syncwarp();
  if (lane < T) {
    const uint32_t fr = P.q_slot_field[(size_t)q * SM + lane];
    const uint32_t f = fr & 0x7Fu;
    const uint32_t ord = P.q_slot_term[(size_t)q * SM + lane];
    PSeg G; memset(&G, 0, sizeof(G)); G.S = P.fields[f].S; G.a128 = P.fields[f].a128; G.t_aoff = P.fields[f].t_aoff; G.n_terms = P.fields[f].n_terms;
    OTerm c = pl_term(G, ord == SB200_NO_TERM ? 0xFFFFFFFFu : ord);
    c.weight = P.q_idf[(size_t)q * SM + lane];
    tc[lane] = c; s_wf[lane] = P.q_idf_f[(size_t)q * SM + lane]; s_fld[lane] = fr;
    s_cur[lane] = 0; s_cached[lane] = 0xFFFFFFFFu;
    if (!(fr & 0x80u)) atomicAdd(s_nf + f, 1u);   // num_query_terms counts text slots only
  }
  __syncwarp();
  bool bad = false;
  uint32_t tf[TMAX];
  uint32_t k = 0, n_slots[2] = {0, 0};   // warp-uniform: distance slots so far, per field
  bool all[2] = {true, true};            // every distance slot of the field holds this lane's document
#pragma unroll
  for (int x = 0; x < TMAX; x++) {
    tf[x] = 0;
    if ((uint32_t)x >= T) continue;
    const uint32_t fld = s_fld[x];       // a rule slot (| 0x80) never equals a field index
    const int df = fld == W.dist[0] ? 0 : (fld == W.dist[1] ? 1 : -1);
    const MField& F = P.fields[fld & 0x7Fu];
    PSeg G; G.S = F.S; G.a128 = F.a128; G.t_aoff = F.t_aoff; G.n_terms = F.n_terms;
    WpPos pos; pos.pre = pre + x * 128; pos.base = df >= 0 ? W.pos_base[df] : nullptr; pos.first = tc[x].first; pos.off = 0;
    const uint64_t r = wp_seek(G, tc[x], s_cur + x, s_cached + x, docs + x * 128, tfs + x * 128, bloom + x * 16, d, live, lane, pos);
    if (r == PL_BAD) bad = true; else tf[x] = (uint32_t)r;
    if (df >= 0) {
      if (live) { W.s_off[(size_t)e * W.nd + k] = pos.off; W.s_tf[(size_t)e * W.nd + k] = tf[x]; }
      k++; n_slots[df]++;
      if (tf[x] == 0) all[df] = false;
    }
  }
  unsigned long long my_work = 0, my_docs = 0;
  if (live) {
    WpSink sink; sink.v = W.o_values + (size_t)at * P.n_ops; sink.s = W.o_scores + (size_t)at * P.n_ops; sink.b = 1.0;
    m_total<TMAX, true>(P, s_ops, s_cache, s_nf, s_fld, s_wf, tc, T, q, d, tf, q, o_nr, sink);
    W.o_boosts[at] = sink.b;
    for (uint32_t f = 0; f < 2; f++) {
      if (n_slots[f] >= 2 && all[f]) {   // decided by the positions
        const unsigned long long i = atomicAdd(W.counters + 0, 1ull);
        W.work[i] = ((unsigned long long)e << 1) | f;
        my_work++;
      } else {                            // an unregistered field, < 2 slots, or a slot without the document: no pair has a b > a
        W.o_slop[(size_t)at * 2 + f] = 0xFFFFFFFFu;
      }
    }
    my_docs = my_work ? 1 : 0;
  }
  for (int o = 16; o; o >>= 1) my_docs += __shfl_down_sync(0xffffffffu, my_docs, o);
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicAdd(W.counters + 1, 1ull);
  if (lane == 0 && my_docs) atomicAdd(W.counters + 2, my_docs);
}

struct WpSlopParams {
  PosView V[2];                             // the distance fields' positions
  uint32_t dist[2];
  const uint64_t* keys; const uint32_t* idx;
  const uint8_t* q_slot_field; const uint32_t* q_slot_term; const uint32_t* q_nslots; uint32_t n_slots_max;
  uint32_t nd; const uint64_t* s_off; const uint32_t* s_tf;
  const unsigned long long* work; unsigned long long n;
  uint32_t* scratch; unsigned long long* scratch_cursor;   // scratch == NULL: shared-memory pass
  unsigned long long* ov_list; unsigned long long* ov;    // items for the global pass; ov[0] = count, ov[1] = their positions
  uint32_t* o_slop;
  unsigned long long* counters;             // [1] format errors [3] positions decoded [4] position bytes
};

__global__ void __launch_bounds__(PH_WARPS * 32) k_wp_slop(const WpSlopParams P) {
  __shared__ __align__(16) uint32_t s_buf[PH_WARPS][PH_SMEM_WORDS];
  __shared__ uint32_t s_tail[PH_WARPS][128];
  __shared__ uint64_t s_o[PH_WARPS][16];
  __shared__ uint32_t s_ord[PH_WARPS][16], s_n[PH_WARPS][16], s_st[PH_WARPS][17];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  unsigned long long n_dec = 0, n_bytes = 0;
  bool bad = false;
  for (unsigned long long it = (unsigned long long)blockIdx.x * PH_WARPS + warp; it < P.n; it += (unsigned long long)gridDim.x * PH_WARPS) {
    const unsigned long long w = P.work[it];
    const uint64_t e = w >> 1;
    const uint32_t f = (uint32_t)(w & 1u);
    const uint32_t q = (uint32_t)(P.keys[e] >> 32);
    const uint32_t T = min(P.q_nslots[q], 16u);
    const uint32_t fld = lane < T ? P.q_slot_field[(size_t)q * P.n_slots_max + lane] : 0xFFu;
    const unsigned md = __ballot_sync(0xffffffffu, lane < T && (fld == P.dist[0] || fld == P.dist[1]));
    const unsigned mf = __ballot_sync(0xffffffffu, lane < T && fld == P.dist[f]);
    if ((mf >> lane) & 1u) {   // the field's slots in slot order; their column in the offset scratch counts both fields
      const uint32_t j = __popc(mf & lt), col = __popc(md & lt);
      s_ord[warp][j] = P.q_slot_term[(size_t)q * P.n_slots_max + lane];
      s_o[warp][j] = P.s_off[e * P.nd + col]; s_n[warp][j] = P.s_tf[e * P.nd + col];
    }
    __syncwarp();
    const uint32_t n = __popc(mf);
    uint64_t S = 0;
    for (uint32_t j = 0; j < n; j++) { s_st[warp][j] = (uint32_t)S; S += s_n[warp][j]; }
    uint32_t* buf;
    if (!P.scratch) {
      if (S > PH_SMEM_WORDS) {
        if (lane == 0) { const unsigned long long i = atomicAdd(P.ov + 0, 1ull); P.ov_list[i] = w; atomicAdd(P.ov + 1, (unsigned long long)S); }
        __syncwarp();
        continue;
      }
      buf = s_buf[warp];
    } else {
      unsigned long long off = 0;
      if (lane == 0) off = atomicAdd(P.scratch_cursor, (unsigned long long)S);
      buf = P.scratch + __shfl_sync(0xffffffffu, off, 0);
    }
    const PosView& V = P.V[f];
    bool ok = true;
    for (uint32_t j = 0; j < n; j++) {
      const uint32_t ord = s_ord[warp][j], tf = s_n[warp][j];
      const uint64_t o = s_o[warp][j];
      if (o + tf > V.count[ord]) { ok = false; break; }   // the skip entries' tf sums disagree with the positions file
      n_bytes += ph_read_deltas(V, ord, o, tf, buf + s_st[warp][j], s_tail[warp], lane);
      ph_prefix(buf + s_st[warp][j], tf, 0u, lane);     // positions_with_offset(0): absolute positions
    }
    if (!ok) { bad = true; __syncwarp(); continue; }
    uint32_t res = 0;
    for (uint32_t j = 0; j + 1 < n; j++) {
      const uint32_t* A = buf + s_st[warp][j]; const uint32_t na = s_n[warp][j];
      const uint32_t* B = buf + s_st[warp][j + 1]; const uint32_t nb = s_n[warp][j + 1];
      uint32_t mine = 0xFFFFFFFFu;
      for (uint32_t i = lane; i < na; i += 32) {
        const uint32_t a = A[i];
        uint32_t lo = 0, hi = nb;   // the smallest b > a
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (B[mid] <= a) lo = mid + 1; else hi = mid; }
        if (lo < nb) mine = min(mine, B[lo] - a);
      }
      res = max(res, __reduce_min_sync(0xffffffffu, mine));
    }
    n_dec += S;
    if (lane == 0) P.o_slop[(size_t)P.idx[e] * 2 + f] = res;
    __syncwarp();
  }
  if (lane == 0) {
    if (bad) atomicAdd(P.counters + 1, 1ull);
    if (n_dec) atomicAdd(P.counters + 3, n_dec);
    if (n_bytes) atomicAdd(P.counters + 4, n_bytes);
  }
}

}  // namespace sb200
