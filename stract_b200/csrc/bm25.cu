// bm25.cu -- hot path 2: BM25 posting-list scoring + top-k on the device (see stract_b200_bm25.h).
//
// Data layout in HBM (per segment/field)
//   postings   the tantivy postings file, byte for byte                       ~1.0-1.5 B / posting
//   fieldnorm  1 byte per doc (FieldNormReader)                               1 B / doc
//   directory  built once from the skip lists: per 128-doc block {last_doc u32, byte offset u32,
//              bit widths u16}; per term {data offset, end offset, doc_freq, first block slot}
//   signals    optional row-major [max_doc][n_cols] f64 numeric signal scores (one 32-B sector per doc at 4 cols)
//
// Which kernel serves which batch (all exhaustive, exact top-k, scores in the reference's f32/f64 operation order):
//   AND                  k_and3 + k_and3_select (bm25_and3.cuh): one warp per (query, 4 blocks of its rarest clause)
//                        appends the hits to a candidate list, the select kernel takes the top-k per query.
//   OR, signal combine   k_or3<MODE, TMAX> (bm25_or3.cuh): one warp per work item walks the terms' posting lists
//                        block-synchronously with TMA staging; TMAX is the smallest of 2/3/5/8 covering the batch.
//   k_topk_warp<MODE> (bm25_warp.cuh), the same walk without k_or3's specialisations, takes the two batches the kernels
//   above do not:
//     * AND with a single-clause query above 65 536 postings: every posting of it is a hit, so k_and3's candidate
//       list would be the whole posting list and the select pass would crawl through it;
//     * signal combine with max_docs: k_or3 has no max_docs short circuit.
//   Block-WAND replay    k_wand (bm25_wand.cuh), one warp per query in the reference's pruning and summation order.
//   multi-field signals  k_sig_multi<TMAX> (bm25_multi.cuh).
//   phrases              k_phrase_cand + k_phrase_verify + k_and3_select (bm25_phrase.cuh).
//   optic pattern docsets k_phrase_cand + k_pattern_verify and word kernels (bm25_pattern.cuh); k_sig_multi<TMAX, true>
//                        consumes them in the recall stage.
//   query-plan docsets   k_plan_cover + CUB sort + k_plan_eval + CUB select (bm25_plan.cuh); k_plan_recall scores them.
//   recall webpages      CUB sort + k_wp_signals + k_wp_slop (bm25_webpage.cuh): signals, boosts and term distances of given docs.
// A query of the walk kernels much larger than the batch average is cut into doc-range work items (plan_items);
// k_merge_topk merges their partial top-k lists.  Keys are (order-preserving score bits, ~doc), so the result order
// is the reference's (score desc, doc asc) total order.
// Roofline: HBM by bytes (posting bytes + 1 B fieldnorm (+ 8 B x n_cols signals) per scored doc), but at the
// configured sizes the postings file is L2-resident and the kernels are bound by unpack/search issue rate.
#include "common.cuh"
#include "../../include/stract_b200_bm25.h"

#ifndef SB200_EMU
#include <cub/cub.cuh>
#endif
#include <algorithm>
#include <cstdlib>
#include <vector>

namespace sb200 {
uint32_t fieldnorm_value(uint8_t id);
struct MergeJob { uint32_t first_slot, n_slots, out_slot, _pad; };
}

struct sb200_signals {
  int device = 0;
  uint32_t n_cols = 0, max_doc = 0;
  sb200::DevBuf<double> rows;
};

struct sb200_segment {
  int device = 0, record = 1, stride = 8;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, evk0 = nullptr, evk1 = nullptr;
  uint32_t max_doc = 0, n_terms = 0;
  uint64_t postings_len = 0, n_blocks = 0, n_postings = 0;
  double stage_ms = 0;
  sb200::DevBuf<uint8_t> postings, fieldnorm;
  sb200::DevBuf<uint64_t> t_data_off, t_end_off;
  sb200::DevBuf<uint32_t> t_df, t_first;
  sb200::DevBuf<uint32_t> b_last, b_off;
  sb200::DevBuf<uint16_t> b_bits, b_bw;   // b_bw: the block-wand (fieldnorm id | tf << 8) pair of every skip entry
  std::vector<uint32_t> h_df;  // host copy (query planning: Intersection sorts by size_hint)
  // per-batch scratch (grown on demand)
  sb200::DevBuf<uint32_t> q_terms, q_nterms, o_docs, o_n, q_orig;
  sb200::DevBuf<float> q_weights, q_cache, o_scores;
  sb200::DevBuf<double> o_totals, q_coeffs;
  sb200::DevBuf<unsigned long long> counters;
  // 16-byte aligned copy of every term's block region (blocks are multiples of 16 bytes) for LDG.128 unpacking
  sb200::DevBuf<uint4> a_post;
  sb200::DevBuf<uint64_t> t_aoff;           // per term, in uint4 units
  sb200::DevBuf<uint64_t> g_khi;            // per-query candidate buffers of the warp kernel
  sb200::DevBuf<uint32_t> g_klo;
  sb200::DevBuf<uint32_t> q_items;          // item -> (query slot, lo, hi, output slot), SoA
  sb200::DevBuf<sb200::MergeJob> q_jobs;
  // scratch of the unit-based AND path (bm25_and3.cuh)
  sb200::DevBuf<uint4> a3_units;            // AUnit records
  sb200::DevBuf<uint64_t> a3_off;           // per query slot: start of its candidate list
  sb200::DevBuf<uint32_t> a3_cnt, a3_key, a3_doc;
  // scratch of the multi-field signal path (bm25_multi.cuh); lives in the FIRST field's handle
  sb200::DevBuf<uint8_t> m_fields, m_ops, m_slot_field;
  sb200::DevBuf<float> m_idf_f;
  sb200::DevBuf<double> m_boost;
  // sparse result tables go to the host packed (copy_out_tables)
  sb200::DevBuf<uint32_t> p_docs, p_scores; sb200::DevBuf<uint64_t> p_off;
  uint32_t* h_pack = nullptr; size_t h_pack_words = 0;   // page-locked staging: [n counts | offsets (u64) | docs | scores]
  // positions (sb200_segment_attach_positions, bm25_phrase.cuh)
  bool has_pos = false;
  sb200::DevBuf<uint8_t> pos_file;
  sb200::DevBuf<uint64_t> pos_data_off, pos_tail_off, pos_end_off, pos_count;   // per term
  sb200::DevBuf<uint32_t> pos_first, pos_nblk;                                   // per term
  sb200::DevBuf<uint64_t> pos_b_off; sb200::DevBuf<uint8_t> pos_b_w;            // per positions block
  sb200::DevBuf<uint64_t> pos_base;                                              // per posting block slot
  std::vector<uint64_t> h_pos_count;
  // scratch of the phrase path
  sb200::DevBuf<uint32_t> ph_shift, ph_slop, ph_cdoc, ph_ctf, ph_mcnt, ph_mkey, ph_mdoc, ph_scratch;
  sb200::DevBuf<float> ph_weight;
  sb200::DevBuf<uint64_t> ph_coff, ph_pre;
  sb200::DevBuf<unsigned long long> ph_ov, ph_ovc;
  // token-count fast field of the field (sb200_segment_attach_token_counts, bm25_pattern.cuh)
  bool has_tok = false;
  sb200::DevBuf<uint64_t> tok_count;
  // scratch of the pattern path and of the optic recall stage (the latter in the first field's handle)
  sb200::DevBuf<uint32_t> pt_col, pt_nparts; sb200::DevBuf<uint8_t> pt_parts; sb200::DevBuf<uint64_t> pt_bits;
  sb200::DevBuf<uint64_t> o_bits; sb200::DevBuf<uint32_t> o_nrules, o_rule, o_exclude, o_require; sb200::DevBuf<double> o_boost;
  // scratch of the plan docset stage (bm25_plan.cuh; in the first plan segment's handle)
  sb200::DevBuf<uint8_t> pl_segs, pl_nodes, pl_cover, pl_keep, pl_tmp;
  sb200::DevBuf<uint64_t> pl_keys, pl_keys2, pl_beg, pl_cnt;
  sb200::DevBuf<uint32_t> pl_off, pl_units, pl_ph_off, pl_ph_docs;
  // scratch of the recall webpages (bm25_webpage.cuh; in the first field's handle)
  sb200::DevBuf<uint64_t> wp_keys, wp_keys2, wp_off, wp_work, wp_ovl, wp_ovc;
  sb200::DevBuf<uint32_t> wp_idx, wp_idx2, wp_beg, wp_units, wp_tf, wp_slop, wp_scratch;
  sb200::DevBuf<double> wp_values, wp_scores, wp_boosts;
  sb200::DevBuf<uint8_t> wp_tmp;
};

struct sb200_docset {
  int device = 0;
  uint32_t max_doc = 0;
  sb200::DevBuf<uint32_t> bits;   // ceil(max_doc / 32) words
};

namespace sb200 {

constexpr int NT = 128;            // threads per CTA == postings per block
constexpr int MAXT = SB200_MAX_QUERY_TERMS;
constexpr uint32_t TERMINATED = 0x7FFFFFFFu;

struct SegView {
  const uint32_t* p32; uint64_t postings_len;
  const uint8_t* fieldnorm; uint32_t max_doc;
  const uint64_t *t_data_off, *t_end_off; const uint32_t *t_df, *t_first;
  const uint32_t *b_last, *b_off; const uint16_t* b_bits;
  int record;
};

// ------------------------------------------------------------------ directory build -------------
// one warp per term: parse [VInt skip_len] and turn the skip entries into randomly addressable block records
__global__ void k_build_directory(const uint8_t* __restrict__ postings, const sb200_term_info* __restrict__ terms,
                                  uint32_t n_terms, int stride, const uint32_t* __restrict__ t_first,
                                  uint64_t* t_data_off, uint64_t* t_end_off, uint32_t* t_df, uint32_t* b_last,
                                  uint32_t* b_off, uint16_t* b_bits, uint16_t* b_bw, uint64_t postings_len, int* err) {
  const uint32_t t = (blockIdx.x * (uint32_t)blockDim.x + threadIdx.x) >> 5;
  if (t >= n_terms) return;
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t off = terms[t].postings_off, len = terms[t].postings_len;
  const uint32_t df = terms[t].doc_freq;
  const uint32_t nfull = df >> 7, first = t_first[t];
  if (off + len > postings_len) { if (lane == 0) *err = 1; return; }
  uint64_t skip_start = off, skip_len = 0;
  if (df >= 128) {  // split_into_skips_and_postings, block_segment_postings.rs:78-88
    // every read stays inside [off, off + len): the TermInfo is caller data and may be corrupt
    int sh = 0; uint64_t p = off; bool closed = false;
    for (int i = 0; i < 10 && p < off + len; i++) { const uint8_t b = postings[p++]; skip_len |= (uint64_t)(b & 127u) << sh; if (b & 128u) { closed = true; break; } sh += 7; }
    skip_start = p;
    if (!closed || skip_len != (uint64_t)nfull * stride || skip_start + skip_len > off + len) { if (lane == 0) *err = 2; return; }
  }
  const uint64_t data_off = skip_start + skip_len;
  if (lane == 0) { t_data_off[t] = data_off; t_end_off[t] = off + len; t_df[t] = df; }
  uint32_t run = 0;
  for (uint32_t base = 0; base < nfull; base += 32) {
    const uint32_t j = base + lane;
    uint32_t size = 0, last = 0; uint16_t bits = 0, bw = 0;
    if (j < nfull) {
      const uint8_t* e = postings + skip_start + (uint64_t)j * stride;  // skip.rs:186-238
      last = (uint32_t)e[0] | ((uint32_t)e[1] << 8) | ((uint32_t)e[2] << 16) | ((uint32_t)e[3] << 24);
      const uint32_t db = e[4] & 0x3fu, strict = (e[4] >> 6) & 1u;
      const uint32_t tb = (stride >= 8) ? e[5] : 0u;
      bits = (uint16_t)(db | (strict << 6) | (tb << 8));
      size = (db + tb) * 16u;
      if (stride >= 8) { const int o = stride == 12 ? 10 : 6; bw = (uint16_t)(e[o] | ((uint32_t)e[o + 1] << 8)); }   // skip.rs:203-232
      if (db > 32 || tb > 32) *err = 3;
    }
    uint32_t incl = size;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t n = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += n; }
    if (j < nfull) { b_last[first + j] = last; b_bits[first + j] = bits; b_bw[first + j] = bw; b_off[first + j] = run + incl - size; }
    run += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (lane == 0) {
    b_off[first + nfull] = run; b_last[first + nfull] = TERMINATED; b_bits[first + nfull] = 0; b_bw[first + nfull] = 0;
    if (data_off + run > off + len) *err = 4;
  }
}

// ------------------------------------------------------------------ device helpers ---------------
__device__ __forceinline__ uint32_t ord_f32(float f) { const uint32_t b = __float_as_uint(f); return (b & 0x80000000u) ? ~b : (b | 0x80000000u); }
__device__ __forceinline__ float unord_f32(uint32_t o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o); }
// f64 totals order by f64::total_cmp (collector/top_docs.rs:229-233: -0.0 below +0.0, +-inf at the ends), except that every
// NaN is first made the negative quiet NaN 0xFFF8000000000000: a NaN total ranks below -inf whatever sign and payload it
// carries (a NaN column keeps its own through the combine), never meets the (0, 0) padding key, and unord_f64 returns that NaN
__device__ __forceinline__ uint64_t ord_f64(double f) {
  const uint64_t b = f != f ? 0xFFF8000000000000ull : (uint64_t)__double_as_longlong(f);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double unord_f64(uint64_t o) { return __longlong_as_double((long long)((o >> 63) ? (o & 0x7FFFFFFFFFFFFFFFull) : ~o)); }

// first index in the sorted 128-entry block with value >= x (branchless, block_search.rs:23-34)
__device__ __forceinline__ uint32_t lower_bound128(const uint32_t* a, uint32_t x) {
  uint32_t start = 0;
#pragma unroll
  for (uint32_t len = 64; len >= 1; len >>= 1) if (a[start + len - 1] < x) start += len;
  // the 7 halving steps count at most 127 smaller elements (the reference may assume target <= last element,
  // we may not): one more probe makes the result 128 when every element is smaller
  if (a[start] < x) start++;
  return start;
}

__device__ __forceinline__ bool key_gt(uint64_t ah, uint32_t al, uint64_t bh, uint32_t bl) { return ah > bh || (ah == bh && al > bl); }

__global__ void k_interleave_signals(const double* const* cols, uint32_t n_cols, uint32_t max_doc, double* rows) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= (uint64_t)max_doc * n_cols) return;
  const uint32_t d = (uint32_t)(i / n_cols), c = (uint32_t)(i % n_cols);
  rows[i] = cols[c][d];
}

// The numeric CoreSignals' value -> score transforms (core/src/ranking/signals/core/non_text.rs:25-101 and the per-signal
// `compute`), one thread per document, written straight into column `c` of the row-major table.  Every expression is the
// reference's f64 expression with explicitly rounded operations; score_rank (a libm `ln`) is not here -- see the host side.
__global__ void k_numeric_score(uint32_t kind, uint32_t dtype, const void* __restrict__ raw, uint32_t max_doc, double p0, double p1,
                                const double* __restrict__ lut, uint32_t lut_len, double* __restrict__ rows, uint32_t n_cols, uint32_t c) {
  const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= max_doc) return;
  unsigned long long u = 0; double f = 0.0;
  if (dtype == SB200_NUM_F64) f = ((const double*)raw)[d];
  else if (dtype == SB200_NUM_U64) { u = ((const unsigned long long*)raw)[d]; f = __ull2double_rn(u); }
  else { u = ((const uint8_t*)raw)[d] ? 1ull : 0ull; f = (double)u; }
  double s = 0.0;
  switch (kind) {
    case SB200_NUM_IDENTITY: s = f; break;                                                   // HostCentrality, PageCentrality (:117-155, :203-241)
    case SB200_NUM_BOOL: s = u ? 1.0 : 0.0; break;                                           // IsHomepage (:289-332)
    case SB200_NUM_BOOL_NOT: s = u ? 0.0 : 1.0; break;                                       // HasAds: score = !has_ads (:730-771)
    case SB200_NUM_INVERSE: s = __ddiv_rn(1.0, __dadd_rn(f, 1.0)); break;                    // score_trackers / digits / slashes (:61-74)
    case SB200_NUM_FETCH_TIME: s = u >= 1000ull ? 0.0 : __ddiv_rn(1.0, __dadd_rn(f, 1.0)); break;   // fetch_time_ms_cache (computer/mod.rs:257-259)
    case SB200_NUM_UPDATE_TIME: {                                                            // score_timestamp (:25-42) over update_time_cache
      const unsigned long long now = (unsigned long long)p0;                                 //   (computer/mod.rs:261-265), 72 / (hours + 72)
      if (u < now) {
        unsigned long long secs = now - u; if (secs < 1ull) secs = 1ull;
        const unsigned long long hours = secs / 3600ull;
        if (hours < 3ull * 365ull * 24ull) s = __ddiv_rn(72.0, __dadd_rn(__ull2double_rn(hours), 72.0));
      }
      break;
    }
    case SB200_NUM_LINK_DENSITY: s = f > 0.5 ? 0.0 : __dsub_rn(1.0, f); break;               // score_link_density (:76-83)
    case SB200_NUM_REGION: {                                                                 // score_region (:85-101): boost + count / total
      if (lut) {                                                                             //   lut absent = no RegionCount: the signal is 0
        const double boost = (p1 != 0.0 && u == (unsigned long long)p0) ? 50.0 : 0.0;         //   p1: a region other than All is selected, p0: its id
        s = __dadd_rn(boost, u < lut_len ? lut[u] : 0.0);
      }
      break;
    }
    default: break;
  }
  rows[(size_t)d * n_cols + c] = s;
}

template <class T>
static int ensure(DevBuf<T>& b, size_t n) { if (b.n < n) return b.alloc(n + (n >> 2) + 16); return SB200_OK; }

}  // namespace sb200
#include "tma.cuh"
#include "bm25_warp.cuh"
namespace sb200 {

template <int MODE>
static int launch_topk_warp(const WParams& P, cudaStream_t s) {
  const size_t per_warp = (size_t)P.n_terms_max * 128 * 8 + sizeof(WTerm) * P.n_terms_max + 32 * 4;
  const size_t sm = 1024 + WQ * per_warp;
  static size_t configured[3] = {0, 0, 0};
  if (sm > 48 * 1024 && configured[MODE] < sm) {
    SB_CUDA(cudaFuncSetAttribute(k_topk_warp<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    configured[MODE] = sm;
  }
  SB_LAUNCH(k_topk_warp<MODE>, div_up(P.n_items, WQ), WQ * 32, sm, s, P);
  SB_CHECK_LAUNCH();
  return SB200_OK;
}

}  // namespace sb200
#include "bm25_and3.cuh"
#include "bm25_or3.cuh"
#include "bm25_multi.cuh"
#include "bm25_wand.cuh"
#include "bm25_phrase.cuh"
#include "bm25_pattern.cuh"
#include "bm25_plan.cuh"
#include "bm25_webpage.cuh"
#include <chrono>
#include <functional>
namespace sb200 {

static void seg_view(const sb200_segment* g, SegView& S) {
  S.p32 = (const uint32_t*)g->postings.p; S.postings_len = g->postings_len; S.fieldnorm = g->fieldnorm.p; S.max_doc = g->max_doc;
  S.t_data_off = g->t_data_off.p; S.t_end_off = g->t_end_off.p; S.t_df = g->t_df.p; S.t_first = g->t_first.p;
  S.b_last = g->b_last.p; S.b_off = g->b_off.p; S.b_bits = g->b_bits.p; S.record = g->record;
}

// Work items of a batch whose query slots are ordered by decreasing work: a query much larger than the average is cut
// into <= 16 doc ranges (W*k <= 16384 for the merge); their partial top-k lists are merged by k_merge_topk.
struct ItemPlan {
  std::vector<uint32_t> q, lo, hi, out;
  std::vector<MergeJob> jobs;
  uint32_t extra = 0, capm = 0;
};
static void plan_items(const std::vector<uint64_t>& work, const std::vector<uint32_t>& order, uint32_t k, uint32_t max_doc, bool can_split, ItemPlan& pl) {
  const uint32_t nq = (uint32_t)work.size();
  uint64_t total = 0;
  for (uint64_t w : work) total += w;
  const uint64_t target = std::max<uint64_t>(32768, total / std::max<uint32_t>(nq, 1));
  const uint32_t wmax = std::max<uint32_t>(1, std::min<uint32_t>(16, 16384 / k));
  for (uint32_t slot = 0; slot < nq; slot++) {
    uint32_t W = can_split ? (uint32_t)std::min<uint64_t>(wmax, (work[slot] + target - 1) / target) : 1;
    if (W < 1) W = 1;
    if (W == 1) { pl.q.push_back(slot); pl.lo.push_back(0); pl.hi.push_back(0xFFFFFFFFu); pl.out.push_back(order[slot]); continue; }
    MergeJob j; j.first_slot = nq + pl.extra; j.n_slots = W; j.out_slot = order[slot]; j._pad = 0;
    pl.jobs.push_back(j);
    for (uint32_t c = 0; c < W; c++) {
      pl.q.push_back(slot);
      pl.lo.push_back((uint32_t)((uint64_t)max_doc * c / W));
      pl.hi.push_back(c + 1 == W ? 0xFFFFFFFFu : (uint32_t)((uint64_t)max_doc * (c + 1) / W));
      pl.out.push_back(nq + pl.extra + c);
    }
    pl.extra += W;
  }
  if (!pl.jobs.empty()) { pl.capm = 1024; while (pl.capm < wmax * k) pl.capm <<= 1; }
}

template <int TMAX, bool OPTIC>
static int launch_multi(const MParams& P, cudaStream_t s) {
  const size_t sm = m_cta_smem<TMAX>();
  static bool configured = false;
  if (!configured) { SB_CUDA(cudaFuncSetAttribute(k_sig_multi<TMAX, OPTIC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm)); configured = true; }
  SB_LAUNCH((k_sig_multi<TMAX, OPTIC>), div_up(P.n_items, WQ), WQ * 32, sm, s, P);
  SB_CHECK_LAUNCH();
  return SB200_OK;
}

typedef std::function<int(uint32_t g0, uint32_t g1, const uint64_t* keys, const uint64_t* q_beg, const std::vector<uint64_t>& h_beg)> PlanEmit;
static int run_plan(const sb200_recall_plan_batch* pb, PlanEmit emit, sb200_plan_stats* stats);
template <int TMAX>
static int launch_plan_recall(const PlanRecallParams& R, cudaStream_t s) {
  const size_t sm = pl_cta_smem<TMAX>();
  static bool configured = false;
  if (!configured) { SB_CUDA(cudaFuncSetAttribute(k_plan_recall<TMAX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm)); configured = true; }
  SB_LAUNCH(k_plan_recall<TMAX>, div_up(R.M.n_queries, WQ), WQ * 32, sm, s, R);
  SB_CHECK_LAUNCH();
  return SB200_OK;
}

struct WpCall { const sb200_webpage_batch* b; const sb200_webpage_out* out; sb200_webpage_stats* stats; };
static int run_webpages(sb200_segment* g, const MParams& P, const sb200_multi_signal_batch* b, const std::vector<uint8_t>& sf,
                        const std::vector<uint32_t>& ns, const WpCall& wp);

// pb != NULL: the candidates are each query's plan docset (run_plan) instead of the union of its text slots.  wp != NULL: no
// top-k; the signals, boosts and term distances of the caller's documents (run_webpages).
static int run_multi(const sb200_multi_signal_batch* b, const sb200_optic_batch* ob, uint32_t* docs, double* totals, uint32_t* n_out,
                     sb200_bm25_stats* stats, const sb200_recall_plan_batch* pb = nullptr, const WpCall* wp = nullptr) {
  if (!b || !b->fields || !b->ops || !b->slot_field || !b->slot_term || !b->slot_idf || !b->slot_idf_f || (!wp && (!docs || !totals || !n_out)))
    SB_FAIL(SB200_EINVAL, "NULL argument");
  const uint32_t nq = b->n_queries, SM = b->n_slots, k = b->k, NF = b->n_fields, NO = b->n_ops;
  if (NF == 0 || NF > (uint32_t)M_MAX_FIELDS) SB_FAIL(SB200_ERANGE, "n_fields %u outside [1,%d]", NF, M_MAX_FIELDS);
  if (NO == 0 || NO > (uint32_t)M_MAX_OPS) SB_FAIL(SB200_ERANGE, "n_ops %u outside [1,%d]", NO, M_MAX_OPS);
  if (SM == 0 || SM > 16) SB_FAIL(SB200_ERANGE, "n_slots %u outside [1,16]", SM);
  if (!wp && (k == 0 || k > SB200_MAX_K)) SB_FAIL(SB200_ERANGE, "k %u outside [1,%d]", k, SB200_MAX_K);
  sb200_segment* g = b->fields[0].seg;
  if (!g) SB_FAIL(SB200_EINVAL, "field 0 has no segment");
  SB_CUDA(cudaSetDevice(g->device));
  cudaStream_t s = g->stream;
  for (uint32_t f = 0; f < NF; f++) {
    const sb200_segment* x = b->fields[f].seg;
    if (!x || !b->fields[f].tf_cache256) SB_FAIL(SB200_EINVAL, "field %u: NULL segment or cache", f);
    if (x->device != g->device || x->max_doc != g->max_doc) SB_FAIL(SB200_EINVAL, "field %u is not a field of the same segment (device / max_doc differ)", f);
  }
  uint32_t n_cols = 0;
  for (uint32_t o = 0; o < NO; o++) {
    const sb200_signal_op& op = b->ops[o];
    if (op.kind > 4u) SB_FAIL(SB200_EINVAL, "op %u: kind %u", o, op.kind);
    if (op.kind != 4u && op.kind != 1u && op.field >= NF) SB_FAIL(SB200_EINVAL, "op %u: field %u >= %u", o, op.field, NF);
    if (op.kind == 4u) {
      if (!b->signals || op.col >= b->signals->n_cols) SB_FAIL(SB200_EINVAL, "op %u: numeric column %u not in the signal table", o, op.col);
      n_cols = b->signals->n_cols;
    }
  }
  if (n_cols && b->signals->max_doc < g->max_doc) SB_FAIL(SB200_EINVAL, "signal table covers %u docs, segment has %u", b->signals->max_doc, g->max_doc);
  if (pb) {
    if (pb->n_queries != nq) SB_FAIL(SB200_EINVAL, "plan batch has %u queries, signal batch %u", pb->n_queries, nq);
    if (!pb->segments || pb->n_segments == 0) SB_FAIL(SB200_EINVAL, "plan batch without segments");
    for (uint32_t i = 0; i < pb->n_segments; i++) {
      const sb200_segment* x = pb->segments[i];
      if (!x || x->device != g->device || x->max_doc != g->max_doc) SB_FAIL(SB200_EINVAL, "plan segment %u is not a field of the signal fields' segment (device / max_doc differ)", i);
    }
  }
  if (ob) {   // optic docsets: shapes, indices, devices; rule slots and docset rules never share a query
    if (ob->n_docsets && !ob->docsets) SB_FAIL(SB200_EINVAL, "optic: NULL docsets");
    if (ob->n_rules && (!ob->rule_docset || !ob->rule_boost)) SB_FAIL(SB200_EINVAL, "optic: NULL rule_docset / rule_boost");
    if (ob->n_rules && (ob->max_rules == 0 || ob->max_rules > SB200_MAX_OPTIC_RULES)) SB_FAIL(SB200_ERANGE, "optic: max_rules %u outside [1,%d]", ob->max_rules, SB200_MAX_OPTIC_RULES);
    for (uint32_t i = 0; i < ob->n_docsets; i++) {
      const sb200_docset* d = ob->docsets[i];
      if (!d) SB_FAIL(SB200_EINVAL, "optic: docset %u is NULL", i);
      if (d->max_doc != g->max_doc || d->device != g->device) SB_FAIL(SB200_EINVAL, "optic: docset %u has max_doc %u on device %d, the segment %u on %d", i, d->max_doc, d->device, g->max_doc, g->device);
    }
    for (uint32_t q = 0; q < nq; q++) {
      const uint32_t nr = ob->n_rules ? ob->n_rules[q] : 0u;
      if (nr > ob->max_rules || nr > SB200_MAX_OPTIC_RULES) SB_FAIL(SB200_ERANGE, "optic: query %u has %u rules (max %u)", q, nr, std::min<uint32_t>(ob->max_rules, SB200_MAX_OPTIC_RULES));
      for (uint32_t r = 0; r < nr; r++) if (ob->rule_docset[(size_t)q * ob->max_rules + r] >= ob->n_docsets) SB_FAIL(SB200_EINVAL, "optic: query %u rule %u: docset index out of range", q, r);
      for (const uint32_t* f : {ob->exclude, ob->require}) if (f && f[q] != SB200_NO_DOCSET && f[q] >= ob->n_docsets) SB_FAIL(SB200_EINVAL, "optic: query %u: filter docset index out of range", q);
      if (nr) for (uint32_t x = 0; x < SM; x++) {
        const uint8_t f = b->slot_field[(size_t)q * SM + x];
        if (f != 0xFF && (f & 0x80)) SB_FAIL(SB200_EINVAL, "optic: query %u mixes rule slots and docset rules (their order would be undefined)", q);
      }
    }
  }
  if (nq == 0) return SB200_OK;
  // planning: slots keep their query order (the f32 sums depend on it); padding slots (field 0xFF) are dropped
  std::vector<uint8_t> sf((size_t)nq * SM, 0);
  std::vector<uint32_t> st((size_t)nq * SM, SB200_NO_TERM), ns(nq, 0), order(nq);
  std::vector<float> w1((size_t)nq * SM, 0.f), w2((size_t)nq * SM, 0.f);
  std::vector<double> wb(b->slot_boost ? (size_t)nq * SM : 0, 0.0);
  std::vector<uint64_t> work(nq, 0), work_sorted(nq, 0);
  unsigned long long postings = 0;
  for (uint32_t q = 0; q < nq; q++) {
    order[q] = q;
    for (uint32_t x = 0; x < SM; x++) {
      const uint8_t f = b->slot_field[(size_t)q * SM + x];
      if (f == 0xFF) continue;
      if ((f & 0x7F) >= NF) SB_FAIL(SB200_EINVAL, "query %u slot %u: field %u >= %u", q, x, (unsigned)(f & 0x7F), NF);
      if ((f & 0x80) && !b->slot_boost) SB_FAIL(SB200_EINVAL, "query %u slot %u is a rule slot but slot_boost is NULL", q, x);
      const uint32_t ord = b->slot_term[(size_t)q * SM + x];
      if (ord != SB200_NO_TERM && ord < b->fields[f & 0x7F].seg->n_terms) work[q] += b->fields[f & 0x7F].seg->h_df[ord];
    }
    postings += work[q];
  }
  if (!pb && !wp) std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t c) { return work[a] > work[c]; });
  for (uint32_t slot = 0; slot < nq; slot++) {
    const uint32_t q = order[slot];
    uint32_t c = 0;
    for (int pass = 0; pass < 2; pass++)   // text slots first (query order kept), rule docsets behind them (rule order kept)
      for (uint32_t x = 0; x < SM; x++) {
        const uint8_t f = b->slot_field[(size_t)q * SM + x];
        if (f == 0xFF || ((f & 0x80) != 0) != (pass == 1)) continue;
        const size_t o = (size_t)slot * SM + c;
        sf[o] = f; st[o] = b->slot_term[(size_t)q * SM + x]; w1[o] = b->slot_idf[(size_t)q * SM + x]; w2[o] = b->slot_idf_f[(size_t)q * SM + x];
        if (b->slot_boost) wb[o] = b->slot_boost[(size_t)q * SM + x];
        c++;
      }
    ns[slot] = c; work_sorted[slot] = work[q];
  }
  ItemPlan pl;   // the plan path has its own work items (one per query, k_plan_recall) and candidate buffers
  if (!pb && !wp) plan_items(work_sorted, order, k, g->max_doc, true, pl);
  const uint32_t n_items = (uint32_t)pl.q.size();
  const size_t n_slots_out = (size_t)nq + pl.extra;
  uint32_t cap = 1024; while (cap < k + SM * 128u) cap <<= 1;
  // device copies
  std::vector<MField> hf(NF);
  for (uint32_t f = 0; f < NF; f++) {
    memset(&hf[f], 0, sizeof(MField));
    const sb200_segment* x = b->fields[f].seg;
    seg_view(x, hf[f].S); hf[f].a128 = x->a_post.p; hf[f].t_aoff = x->t_aoff.p;
    memcpy(hf[f].cache, b->fields[f].tf_cache256, 256 * 4);
    hf[f].k1p1 = b->fields[f].k1 + 1.0f; hf[f].coef = b->fields[f].bm25f_coefficient; hf[f].n_terms = x->n_terms;
  }
  std::vector<MOp> ho(NO);
  for (uint32_t o = 0; o < NO; o++) { ho[o].kind = b->ops[o].kind; ho[o].field = b->ops[o].field; ho[o].chain = b->ops[o].chain; ho[o].col = b->ops[o].col; ho[o].coeff = b->ops[o].coeff; }
  SB_TRY(ensure(g->m_fields, NF * sizeof(MField))); SB_TRY(ensure(g->m_ops, NO * sizeof(MOp))); SB_TRY(ensure(g->m_slot_field, (size_t)nq * SM));
  SB_TRY(ensure(g->q_terms, (size_t)nq * SM)); SB_TRY(ensure(g->q_weights, (size_t)nq * SM)); SB_TRY(ensure(g->m_idf_f, (size_t)nq * SM));
  SB_TRY(ensure(g->q_nterms, nq)); SB_TRY(ensure(g->q_orig, nq)); SB_TRY(ensure(g->o_docs, n_slots_out * k)); SB_TRY(ensure(g->o_n, n_slots_out));
  SB_TRY(ensure(g->o_totals, n_slots_out * k)); SB_TRY(ensure(g->counters, 4));
  SB_TRY(ensure(g->q_items, (size_t)4 * n_items)); SB_TRY(ensure(g->q_jobs, pl.jobs.size() + 1));
  SB_TRY(ensure(g->g_khi, (size_t)n_items * cap)); SB_TRY(ensure(g->g_klo, (size_t)n_items * cap));
  SB_CUDA(cudaEventRecord(g->ev0, s));
  SB_CUDA(cudaMemcpyAsync(g->m_fields.p, hf.data(), NF * sizeof(MField), cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->m_ops.p, ho.data(), NO * sizeof(MOp), cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->m_slot_field.p, sf.data(), sf.size(), cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_terms.p, st.data(), st.size() * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_weights.p, w1.data(), w1.size() * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->m_idf_f.p, w2.data(), w2.size() * 4, cudaMemcpyHostToDevice, s));
  if (b->slot_boost) { SB_TRY(ensure(g->m_boost, wb.size())); SB_CUDA(cudaMemcpyAsync(g->m_boost.p, wb.data(), wb.size() * 8, cudaMemcpyHostToDevice, s)); }
  SB_CUDA(cudaMemcpyAsync(g->q_nterms.p, ns.data(), ns.size() * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_orig.p, order.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_items.p, pl.q.data(), (size_t)n_items * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_items.p + n_items, pl.lo.data(), (size_t)n_items * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_items.p + 2 * (size_t)n_items, pl.hi.data(), (size_t)n_items * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_items.p + 3 * (size_t)n_items, pl.out.data(), (size_t)n_items * 4, cudaMemcpyHostToDevice, s));
  if (!pl.jobs.empty()) SB_CUDA(cudaMemcpyAsync(g->q_jobs.p, pl.jobs.data(), pl.jobs.size() * sizeof(MergeJob), cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemsetAsync(g->counters.p, 0, 4 * sizeof(unsigned long long), s));
  MParams P;
  memset(&P, 0, sizeof(P));
  P.fields = (const MField*)g->m_fields.p; P.n_fields = NF; P.max_doc = g->max_doc;
  P.ops = (const MOp*)g->m_ops.p; P.n_ops = NO;
  P.q_slot_field = g->m_slot_field.p; P.q_slot_term = g->q_terms.p; P.q_idf = g->q_weights.p; P.q_idf_f = g->m_idf_f.p; P.q_nslots = g->q_nterms.p;
  P.q_boost = b->slot_boost ? g->m_boost.p : nullptr;
  P.q_orig = g->q_orig.p; P.n_queries = nq; P.n_slots_max = SM; P.k = k; P.cap = cap;
  P.n_items = n_items; P.item_q = g->q_items.p; P.item_lo = g->q_items.p + n_items; P.item_hi = g->q_items.p + 2 * (size_t)n_items; P.item_out = g->q_items.p + 3 * (size_t)n_items;
  if (n_cols) { P.sig = b->signals->rows.p; P.n_cols = n_cols; }
  P.g_khi = g->g_khi.p; P.g_klo = g->g_klo.p; P.o_docs = g->o_docs.p; P.o_totals = g->o_totals.p; P.o_n = g->o_n.p; P.counters = g->counters.p;
  std::vector<uint64_t> bp; std::vector<uint32_t> nr, ex, rq, rd; std::vector<double> rb;   // optic tables, alive until the sync
  if (ob) {
    bp.assign(std::max<uint32_t>(ob->n_docsets, 1), 0);
    for (uint32_t i = 0; i < ob->n_docsets; i++) bp[i] = (uint64_t)(uintptr_t)ob->docsets[i]->bits.p;
    const uint32_t MR = ob->n_rules ? ob->max_rules : 1u;
    nr.assign(nq, 0); ex.assign(nq, SB200_NO_DOCSET); rq.assign(nq, SB200_NO_DOCSET); rd.assign((size_t)nq * MR, 0); rb.assign((size_t)nq * MR, 0.0);
    for (uint32_t q = 0; q < nq; q++) {
      nr[q] = ob->n_rules ? ob->n_rules[q] : 0u;
      if (ob->exclude) ex[q] = ob->exclude[q];
      if (ob->require) rq[q] = ob->require[q];
      for (uint32_t r = 0; r < nr[q]; r++) { rd[(size_t)q * MR + r] = ob->rule_docset[(size_t)q * MR + r]; rb[(size_t)q * MR + r] = ob->rule_boost[(size_t)q * MR + r]; }
    }
    SB_TRY(ensure(g->o_bits, bp.size())); SB_TRY(ensure(g->o_nrules, nq)); SB_TRY(ensure(g->o_exclude, nq)); SB_TRY(ensure(g->o_require, nq));
    SB_TRY(ensure(g->o_rule, rd.size())); SB_TRY(ensure(g->o_boost, rb.size()));
    SB_CUDA(cudaMemcpyAsync(g->o_bits.p, bp.data(), bp.size() * 8, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(g->o_nrules.p, nr.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(g->o_exclude.p, ex.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(g->o_require.p, rq.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(g->o_rule.p, rd.data(), rd.size() * 4, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(g->o_boost.p, rb.data(), rb.size() * 8, cudaMemcpyHostToDevice, s));
    P.d_bits = (const uint32_t* const*)g->o_bits.p; P.d_nrules = g->o_nrules.p; P.d_rule = g->o_rule.p; P.d_boost = g->o_boost.p;
    P.d_max_rules = MR; P.d_exclude = g->o_exclude.p; P.d_require = g->o_require.p;
  }
  if (wp) return run_webpages(g, P, b, sf, ns, *wp);
  if (pb) {   // the plan docset group by group; each group's recall runs on this stream once its docset is complete
    SB_CUDA(cudaStreamSynchronize(s));
    uint32_t rcap = 1024; while (rcap < k + 32) rcap <<= 1;
    float kms = 0.0f; unsigned long long scored = 0;
    sb200_plan_stats ps;
    bool restored = false;
    auto emit = [&](uint32_t g0, uint32_t g1, const uint64_t* keys, const uint64_t* q_beg, const std::vector<uint64_t>&) -> int {
      const uint32_t n = g1 - g0;
      if (!restored) {
        // phrase leaves on this handle's field ran the phrase path on it, which reuses (and may have regrown) its term, weight,
        // count and counter scratch: upload the slots again and point the parameters at the current buffers
        SB_TRY(ensure(g->q_terms, st.size())); SB_TRY(ensure(g->q_weights, w1.size())); SB_TRY(ensure(g->q_nterms, ns.size())); SB_TRY(ensure(g->counters, 4));
        SB_CUDA(cudaMemcpyAsync(g->q_terms.p, st.data(), st.size() * 4, cudaMemcpyHostToDevice, s));
        SB_CUDA(cudaMemcpyAsync(g->q_weights.p, w1.data(), w1.size() * 4, cudaMemcpyHostToDevice, s));
        SB_CUDA(cudaMemcpyAsync(g->q_nterms.p, ns.data(), ns.size() * 4, cudaMemcpyHostToDevice, s));
        SB_CUDA(cudaMemsetAsync(g->counters.p, 0, 4 * sizeof(unsigned long long), s));
        P.q_slot_term = g->q_terms.p; P.q_idf = g->q_weights.p; P.q_nslots = g->q_nterms.p; P.counters = g->counters.p;
        restored = true;
      }
      SB_TRY(ensure(g->g_khi, (size_t)n * rcap)); SB_TRY(ensure(g->g_klo, (size_t)n * rcap));
      PlanRecallParams R;
      R.M = P;
      R.M.q_slot_field = P.q_slot_field + (size_t)g0 * SM; R.M.q_slot_term = P.q_slot_term + (size_t)g0 * SM;
      R.M.q_idf = P.q_idf + (size_t)g0 * SM; R.M.q_idf_f = P.q_idf_f + (size_t)g0 * SM; R.M.q_nslots = P.q_nslots + g0;
      if (P.q_boost) R.M.q_boost = P.q_boost + (size_t)g0 * SM;
      R.M.q_orig = P.q_orig + g0; R.M.n_queries = n; R.M.cap = rcap; R.M.g_khi = g->g_khi.p; R.M.g_klo = g->g_klo.p;
      R.keys = keys; R.q_beg = q_beg;
      SB_CUDA(cudaEventRecord(g->evk0, s));
      if (SM <= 8) SB_TRY(launch_plan_recall<8>(R, s)); else SB_TRY(launch_plan_recall<16>(R, s));
      SB_CUDA(cudaEventRecord(g->evk1, s));
      SB_CUDA(cudaStreamSynchronize(s));
      float ms = 0.0f; cudaEventElapsedTime(&ms, g->evk0, g->evk1); kms += ms;
      return SB200_OK;
    };
    SB_TRY(run_plan(pb, emit, &ps));
    SB_CUDA(cudaMemcpyAsync(docs, g->o_docs.p, (size_t)nq * k * 4, cudaMemcpyDefault, s));
    SB_CUDA(cudaMemcpyAsync(totals, g->o_totals.p, (size_t)nq * k * 8, cudaMemcpyDefault, s));
    SB_CUDA(cudaMemcpyAsync(n_out, g->o_n.p, (size_t)nq * 4, cudaMemcpyDefault, s));
    unsigned long long h[4] = {0, 0, 0, 0};
    SB_CUDA(cudaMemcpyAsync(h, g->counters.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaEventRecord(g->ev1, s));
    SB_CUDA(cudaStreamSynchronize(s));
    if (h[2]) SB_FAIL(SB200_EFORMAT, "%llu queries met inconsistent posting data in the plan recall", h[2]);
    scored = h[0];
    if (stats) {
      float ms = 0; cudaEventElapsedTime(&ms, g->ev0, g->ev1);
      stats->postings_scored = postings; stats->docs_scored = scored; stats->blocks_decoded = 0; stats->ms = ms; stats->kernel_ms = kms + ps.kernel_ms;
    }
    return SB200_OK;
  }
  SB_CUDA(cudaEventRecord(g->evk0, s));
  if (ob) { if (SM <= 8) SB_TRY((launch_multi<8, true>(P, s))); else SB_TRY((launch_multi<16, true>(P, s))); }
  else if (SM <= 8) SB_TRY((launch_multi<8, false>(P, s))); else SB_TRY((launch_multi<16, false>(P, s)));
  if (!pl.jobs.empty()) {
    const size_t msm = (size_t)pl.capm * 12;
    static size_t mconf = 0;
    if (msm > 48 * 1024 && mconf < msm) { SB_CUDA(cudaFuncSetAttribute(k_merge_topk<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)msm)); mconf = msm; }
    SB_LAUNCH(k_merge_topk<2>, (unsigned)pl.jobs.size(), 256, msm, s, g->q_jobs.p, k, pl.capm, P.o_docs, (float*)nullptr, P.o_totals, P.o_n);
    SB_CHECK_LAUNCH();
  }
  SB_CUDA(cudaEventRecord(g->evk1, s));
  SB_CUDA(cudaMemcpyAsync(docs, g->o_docs.p, (size_t)nq * k * 4, cudaMemcpyDefault, s));
  SB_CUDA(cudaMemcpyAsync(totals, g->o_totals.p, (size_t)nq * k * 8, cudaMemcpyDefault, s));
  SB_CUDA(cudaMemcpyAsync(n_out, g->o_n.p, (size_t)nq * 4, cudaMemcpyDefault, s));
  unsigned long long h[4] = {0, 0, 0, 0};
  SB_CUDA(cudaMemcpyAsync(h, g->counters.p, sizeof(h), cudaMemcpyDeviceToHost, s));
  SB_CUDA(cudaEventRecord(g->ev1, s));
  SB_CUDA(cudaStreamSynchronize(s));
  if (h[2]) SB_FAIL(SB200_EFORMAT, "%llu queries hit the decode watchdog (inconsistent posting data)", h[2]);
  if (stats) {
    float ms = 0; cudaEventElapsedTime(&ms, g->ev0, g->ev1);
    stats->postings_scored = postings; stats->docs_scored = h[0]; stats->blocks_decoded = h[1]; stats->ms = ms; cudaEventElapsedTime(&stats->kernel_ms, g->evk0, g->evk1);
  }
  return SB200_OK;
}

// union modes through k_or3, instantiated for the smallest term-count bound that covers the batch
template <int MODE>
static int launch_or3(const WParams& P, cudaStream_t s) {
  void (*kern)(const WParams) = k_or3<MODE, 8>;
  if (P.n_terms_max <= 2) kern = k_or3<MODE, 2>;
  else if (P.n_terms_max <= 3) kern = k_or3<MODE, 3>;
  else if (P.n_terms_max <= 5) kern = k_or3<MODE, 5>;
  SB_LAUNCH(kern, div_up(P.n_items, WQ), WQ * 32, 0, s, P);
  SB_CHECK_LAUNCH();
  return SB200_OK;
}

// Result tables to the caller.  An AND batch fills a fraction of its [n_queries][k] table (C4: 72 of 1000 entries per
// query), so the dense copy of 80 MB is mostly padding: when the tables go to host memory and are
// less than half full, the valid prefixes are packed on the device, cross PCIe as one block and are scattered into the
// caller's tables by the host.  f32 scores only (path A); dense copy otherwise.
__global__ void k_pack_tables(const uint32_t* __restrict__ o_n, const uint64_t* __restrict__ off, const uint32_t* __restrict__ o_docs,
                              const float* __restrict__ o_scores, uint32_t k, uint32_t* p_docs, uint32_t* p_scores) {
  const uint32_t q = blockIdx.x, n = o_n[q];
  const uint64_t base = off[q];
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    p_docs[base + i] = o_docs[(size_t)q * k + i];
    p_scores[base + i] = __float_as_uint(o_scores[(size_t)q * k + i]);
  }
}
static int copy_out_tables(sb200_segment* g, uint32_t nq, uint32_t k, uint32_t* docs, float* scores, double* totals, uint32_t* n_out) {
  cudaStream_t s = g->stream;
  const bool sparse_ok = scores && !totals && !is_device_ptr(docs) && !is_device_ptr(scores) && !is_device_ptr(n_out) &&
                         (size_t)nq * k >= (getenv("SB200_BM25_PACK_MIN") ? (size_t)atol(getenv("SB200_BM25_PACK_MIN")) : ((size_t)1 << 18)) &&
                         getenv("SB200_BM25_DENSE_OUT") == nullptr;
  if (sparse_ok) {
    const size_t head = (size_t)nq + 2 * (size_t)nq;   // counts (u32) + offsets (u64 as two words)
    if (g->h_pack_words < head) {
      if (g->h_pack) cudaFreeHost(g->h_pack);
      g->h_pack = nullptr; g->h_pack_words = 0;
      SB_CUDA(cudaMallocHost((void**)&g->h_pack, (head + 1024) * 4));
      g->h_pack_words = head + 1024;
    }
    SB_CUDA(cudaMemcpyAsync(g->h_pack, g->o_n.p, (size_t)nq * 4, cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaStreamSynchronize(s));
    uint64_t total = 0;
    std::vector<uint64_t> off(nq);
    for (uint32_t q = 0; q < nq; q++) { off[q] = total; total += g->h_pack[q]; }
    if (total * 2 < (uint64_t)nq * k) {
      memcpy(n_out, g->h_pack, (size_t)nq * 4);
      if (total == 0) return SB200_OK;
      SB_TRY(ensure(g->p_off, nq)); SB_TRY(ensure(g->p_docs, (size_t)total)); SB_TRY(ensure(g->p_scores, (size_t)total));
      const size_t need = head + 2 * (size_t)total;
      if (g->h_pack_words < need) {
        cudaFreeHost(g->h_pack); g->h_pack = nullptr; g->h_pack_words = 0;
        SB_CUDA(cudaMallocHost((void**)&g->h_pack, (need + (need >> 2)) * 4));
        g->h_pack_words = need + (need >> 2);
      }
      SB_CUDA(cudaMemcpyAsync(g->p_off.p, off.data(), (size_t)nq * 8, cudaMemcpyHostToDevice, s));
      SB_LAUNCH(k_pack_tables, nq, 128, 0, s, g->o_n.p, g->p_off.p, g->o_docs.p, g->o_scores.p, k, g->p_docs.p, g->p_scores.p);
      SB_CHECK_LAUNCH();
      uint32_t* hd = g->h_pack + head; uint32_t* hs = hd + total;
      SB_CUDA(cudaMemcpyAsync(hd, g->p_docs.p, (size_t)total * 4, cudaMemcpyDeviceToHost, s));
      SB_CUDA(cudaMemcpyAsync(hs, g->p_scores.p, (size_t)total * 4, cudaMemcpyDeviceToHost, s));
      SB_CUDA(cudaStreamSynchronize(s));
      for (uint32_t q = 0; q < nq; q++) {
        const uint32_t n = n_out[q];
        if (!n) continue;
        memcpy(docs + (size_t)q * k, hd + off[q], (size_t)n * 4);
        memcpy(scores + (size_t)q * k, hs + off[q], (size_t)n * 4);
      }
      return SB200_OK;
    }
    memcpy(n_out, g->h_pack, (size_t)nq * 4);
    SB_CUDA(cudaMemcpyAsync(docs, g->o_docs.p, (size_t)nq * k * 4, cudaMemcpyDefault, s));
    SB_CUDA(cudaMemcpyAsync(scores, g->o_scores.p, (size_t)nq * k * 4, cudaMemcpyDefault, s));
    return SB200_OK;
  }
  SB_CUDA(cudaMemcpyAsync(docs, g->o_docs.p, (size_t)nq * k * 4, cudaMemcpyDefault, s));
  if (totals) SB_CUDA(cudaMemcpyAsync(totals, g->o_totals.p, (size_t)nq * k * 8, cudaMemcpyDefault, s));
  else if (scores) SB_CUDA(cudaMemcpyAsync(scores, g->o_scores.p, (size_t)nq * k * 4, cudaMemcpyDefault, s));
  SB_CUDA(cudaMemcpyAsync(n_out, g->o_n.p, (size_t)nq * 4, cudaMemcpyDefault, s));
  return SB200_OK;
}

// AND batch through the unit kernel: `terms`/`nterms` are the planned clauses per query slot (sorted by doc_freq),
// results land in g->o_docs / o_scores / o_n at the caller's query index (order[slot]).  Candidate memory is
// sum(doc_freq of the rarest clause) x 8 B; slots are processed in groups that keep it under a budget.
static int run_and3(sb200_segment* g, const SegView& S, const std::vector<uint32_t>& terms, const std::vector<uint32_t>& nterms,
                    uint32_t nq, uint32_t nt, uint32_t k, cudaStream_t s) {
  static_assert(sizeof(AUnit) == sizeof(uint4), "AUnit is stored in a uint4 buffer");
  uint64_t budget = (uint64_t)8 << 30;
  if (const char* e = getenv("SB200_AND3_BUDGET_MB")) { const long mb = atol(e); if (mb > 0) budget = (uint64_t)mb << 20; }
  const uint64_t max_entries = std::max<uint64_t>(budget / 8, 1);
  std::vector<uint64_t> off(nq, 0);
  std::vector<AUnit> units;
  static size_t sel_conf = 0;
  const size_t sel_smem = (size_t)A3_SEL_CAP * 8;
  if (sel_conf < sel_smem) {
    SB_CUDA(cudaFuncSetAttribute(k_and3_select, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sel_smem));
    sel_conf = sel_smem;
  }
  SB_TRY(ensure(g->a3_off, nq)); SB_TRY(ensure(g->a3_cnt, nq));
  uint32_t g0 = 0;
  while (g0 < nq) {
    // group [g0, g1): as many slots as fit the candidate budget (at least one)
    uint64_t entries = 0; uint32_t g1 = g0;
    units.clear();
    while (g1 < nq) {
      const uint32_t dfA = nterms[g1] ? g->h_df[terms[(size_t)g1 * nt]] : 0u;
      if (g1 > g0 && entries + dfA > max_entries) break;
      off[g1] = entries; entries += dfA;
      const uint32_t nblk = (dfA >> 7) + ((dfA & 127u) ? 1u : 0u);
      for (uint32_t b0 = 0; b0 < nblk; b0 += A3_UNIT_BLOCKS) {
        AUnit u; u.q = g1; u.blk_lo = b0; u.blk_hi = std::min(nblk, b0 + A3_UNIT_BLOCKS); u._pad = 0;
        units.push_back(u);
      }
      g1++;
    }
    const uint32_t n_units = (uint32_t)units.size();
    SB_TRY(ensure(g->a3_key, (size_t)std::max<uint64_t>(entries, 1))); SB_TRY(ensure(g->a3_doc, (size_t)std::max<uint64_t>(entries, 1)));
    SB_TRY(ensure(g->a3_units, std::max<size_t>(n_units, 1)));
    if (g0 == 0) SB_CUDA(cudaEventRecord(g->evk0, s));   // kernel_ms starts here: the unit list above is host planning
    SB_CUDA(cudaMemcpyAsync(g->a3_off.p + g0, off.data() + g0, (size_t)(g1 - g0) * 8, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemsetAsync(g->a3_cnt.p + g0, 0, (size_t)(g1 - g0) * 4, s));
    if (n_units) {
      SB_CUDA(cudaMemcpyAsync(g->a3_units.p, units.data(), (size_t)n_units * sizeof(AUnit), cudaMemcpyHostToDevice, s));
      A3Params A;
      memset(&A, 0, sizeof(A));
      A.S = S; A.a128 = g->a_post.p; A.t_aoff = g->t_aoff.p;
      A.q_terms = g->q_terms.p; A.q_nterms = g->q_nterms.p; A.q_weights = g->q_weights.p; A.cache = g->q_cache.p; A.n_terms_max = nt;
      A.units = (const AUnit*)g->a3_units.p; A.n_units = n_units;
      A.cand_off = g->a3_off.p; A.cand_cnt = g->a3_cnt.p; A.c_key = g->a3_key.p; A.c_doc = g->a3_doc.p;
      A.counters = g->counters.p;
      SB_LAUNCH(k_and3, div_up(n_units, A3_WARPS), A3_WARPS * 32, 0, s, A);
      SB_CHECK_LAUNCH();
    }
    SB_LAUNCH(k_and3_select, g1 - g0, 256, sel_smem, s, g->a3_off.p, g->a3_cnt.p, g->a3_key.p, g->a3_doc.p, g->q_orig.p, g0, k,
              g->o_docs.p, g->o_scores.p, g->o_n.p);
    SB_CHECK_LAUNCH();
    if (g1 < nq) SB_CUDA(cudaStreamSynchronize(s));  // `units` / `off` are reused by the next group's async copies
    g0 = g1;
  }
  return SB200_OK;
}

static int run_batch(sb200_segment* g, const sb200_bm25_batch* b, int mode, const sb200_signal_batch* sb, uint32_t* docs,
                     float* scores, double* totals, uint32_t* n_out, sb200_bm25_stats* stats) {
  NvtxRange nvtx(sb ? "sb200 signal top-k batch" : "sb200 bm25 top-k batch");
  cudaStream_t s = g->stream;
  if (!b || !b->term_ords || !b->weights || !b->tf_cache256 || !docs || !n_out) SB_FAIL(SB200_EINVAL, "NULL argument");
  const uint32_t nq = b->n_queries, nt = b->n_terms, k = b->k;
  if (nt == 0 || nt > MAXT) SB_FAIL(SB200_ERANGE, "n_terms %u outside [1,%d]", nt, MAXT);
  if (k == 0 || k > SB200_MAX_K) SB_FAIL(SB200_ERANGE, "k %u outside [1,%d]", k, SB200_MAX_K);
  if (nq == 0) return SB200_OK;
  // host-side planning: drop padding; AND sorts the clauses by doc_freq (stable) like intersect_scorers (intersection.rs:24)
  std::vector<uint32_t> terms((size_t)nq * nt), nterms(nq);
  std::vector<float> weights((size_t)nq * nt);
  unsigned long long postings = 0;
  // longest-processing-time-first: one warp walks a whole query, so the batch finishes when its largest query
  // does; slots are ordered by decreasing posting count and results go back to the caller's index (q_orig)
  std::vector<uint32_t> order(nq);
  std::vector<uint64_t> slot_work(nq, 0);   // postings per query slot
  {
    std::vector<uint64_t> work(nq, 0);
    for (uint32_t q = 0; q < nq; q++) {
      order[q] = q;
      for (uint32_t t = 0; t < nt; t++) { const uint32_t ord = b->term_ords[(size_t)q * nt + t]; if (ord != SB200_NO_TERM && ord < g->n_terms) work[q] += g->h_df[ord]; }
    }
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t bb) { return work[a] > work[bb]; });
  }
  for (uint32_t slot = 0; slot < nq; slot++) {
    const uint32_t q = order[slot];
    uint32_t idx[MAXT]; uint32_t c = 0;
    for (uint32_t t = 0; t < nt; t++) {
      const uint32_t ord = b->term_ords[(size_t)q * nt + t];
      if (ord == SB200_NO_TERM) continue;
      if (ord >= g->n_terms) SB_FAIL(SB200_EINVAL, "query %u: term ordinal %u >= %u", q, ord, g->n_terms);
      idx[c++] = t;
    }
    if (mode == SB200_MODE_AND) std::stable_sort(idx, idx + c, [&](uint32_t a, uint32_t bb) { return g->h_df[b->term_ords[(size_t)q * nt + a]] < g->h_df[b->term_ords[(size_t)q * nt + bb]]; });
    for (uint32_t i = 0; i < c; i++) {
      terms[(size_t)slot * nt + i] = b->term_ords[(size_t)q * nt + idx[i]];
      weights[(size_t)slot * nt + i] = b->weights[(size_t)q * nt + idx[i]];
      slot_work[slot] += g->h_df[terms[(size_t)slot * nt + i]];
    }
    postings += slot_work[slot];
    nterms[slot] = c;
  }
  ItemPlan pl;   // a replayed history (Block-WAND) and the max_docs short circuit cannot be cut into doc ranges
  plan_items(slot_work, order, k, g->max_doc, !(sb && sb->max_docs) && !(!sb && mode == SB200_MODE_OR_WAND), pl);
  const uint32_t n_items = (uint32_t)pl.q.size();
  const size_t n_slots_out = (size_t)nq + pl.extra;
  SB_TRY(ensure(g->q_terms, (size_t)nq * nt)); SB_TRY(ensure(g->q_weights, (size_t)nq * nt)); SB_TRY(ensure(g->q_nterms, nq));
  SB_TRY(ensure(g->q_cache, 256)); SB_TRY(ensure(g->o_docs, n_slots_out * k)); SB_TRY(ensure(g->o_n, n_slots_out));
  if (totals) SB_TRY(ensure(g->o_totals, n_slots_out * k)); else SB_TRY(ensure(g->o_scores, n_slots_out * k));
  SB_TRY(ensure(g->counters, 4)); SB_TRY(ensure(g->q_orig, nq));
  SB_TRY(ensure(g->q_items, (size_t)4 * n_items)); SB_TRY(ensure(g->q_jobs, pl.jobs.size() + 1));
  SB_CUDA(cudaEventRecord(g->ev0, s));
  SB_CUDA(cudaMemcpyAsync(g->q_orig.p, order.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_items.p, pl.q.data(), (size_t)n_items * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_items.p + n_items, pl.lo.data(), (size_t)n_items * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_items.p + 2 * (size_t)n_items, pl.hi.data(), (size_t)n_items * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_items.p + 3 * (size_t)n_items, pl.out.data(), (size_t)n_items * 4, cudaMemcpyHostToDevice, s));
  if (!pl.jobs.empty()) SB_CUDA(cudaMemcpyAsync(g->q_jobs.p, pl.jobs.data(), pl.jobs.size() * sizeof(MergeJob), cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_terms.p, terms.data(), terms.size() * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_weights.p, weights.data(), weights.size() * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_nterms.p, nterms.data(), nterms.size() * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_cache.p, b->tf_cache256, 256 * 4, cudaMemcpyDefault, s));
  SB_CUDA(cudaMemsetAsync(g->counters.p, 0, 4 * sizeof(unsigned long long), s));
  SegView S;
  seg_view(g, S);
  SB_CUDA(cudaEventRecord(g->evk0, s));
  if (!sb && mode != SB200_MODE_AND && mode != SB200_MODE_OR && mode != SB200_MODE_OR_WAND) SB_FAIL(SB200_EINVAL, "mode %d", mode);
  // a single-clause "intersection" makes every posting a hit: its candidate list in k_and3 would be the whole posting list
  // and the select pass would crawl through it chunk by chunk; the threshold-pruning k_topk_warp<AND> handles those batches
  const bool and_long_single = !sb && mode == SB200_MODE_AND && [&] {
    for (uint32_t slot = 0; slot < nq; slot++)
      if (nterms[slot] == 1 && g->h_df[terms[(size_t)slot * nt]] > 65536u) return true;
    return false;
  }();
  if (!sb && mode == SB200_MODE_OR_WAND) {
    // block_wand replayed (bm25_wand.cuh): one warp per query slot, the reference's own pruning and summation order
    if (g->record < 1) SB_FAIL(SB200_EINVAL, "Block-WAND needs term frequencies (record option WithFreqs or above)");
    uint32_t wcap = 2; while (wcap < 2 * k) wcap <<= 1;
    SB_TRY(ensure(g->g_khi, (size_t)nq * wcap)); SB_TRY(ensure(g->g_klo, (size_t)nq * wcap));
    WandParams W;
    memset(&W, 0, sizeof(W));
    W.S = S; W.b_bw = g->b_bw.p; W.a128 = g->a_post.p; W.t_aoff = g->t_aoff.p;
    W.q_terms = g->q_terms.p; W.q_nterms = g->q_nterms.p; W.q_weights = g->q_weights.p; W.cache = g->q_cache.p; W.q_orig = g->q_orig.p;
    W.n_queries = nq; W.n_terms_max = nt; W.k = k; W.cap = wcap;
    W.g_khi = g->g_khi.p; W.g_klo = g->g_klo.p; W.o_docs = g->o_docs.p; W.o_scores = g->o_scores.p; W.o_n = g->o_n.p; W.counters = g->counters.p;
    SB_LAUNCH(k_wand, div_up(nq, WD_WARPS), WD_WARPS * 32, 0, s, W);
    SB_CHECK_LAUNCH();
  } else if (!sb && mode == SB200_MODE_AND && !and_long_single) {
    SB_TRY(run_and3(g, S, terms, nterms, nq, nt, k, s));
  } else {
    // the walk kernels: k_or3 for OR and the signal combine, k_topk_warp for the batches it does not cover
    uint32_t cap = 1024; while (cap < k + nt * 128u) cap <<= 1;
    SB_TRY(ensure(g->g_khi, (size_t)n_items * cap)); SB_TRY(ensure(g->g_klo, (size_t)n_items * cap));
    WParams W;
    memset(&W, 0, sizeof(W));
    W.S = S; W.a128 = g->a_post.p; W.t_aoff = g->t_aoff.p;
    W.q_terms = g->q_terms.p; W.q_nterms = g->q_nterms.p; W.q_weights = g->q_weights.p; W.cache = g->q_cache.p; W.q_orig = g->q_orig.p;
    W.n_queries = nq; W.n_terms_max = nt; W.k = k; W.cap = cap;
    W.n_items = n_items; W.item_q = g->q_items.p; W.item_lo = g->q_items.p + n_items; W.item_hi = g->q_items.p + 2 * (size_t)n_items; W.item_out = g->q_items.p + 3 * (size_t)n_items;
    W.g_khi = g->g_khi.p; W.g_klo = g->g_klo.p;
    W.o_docs = g->o_docs.p; W.o_scores = g->o_scores.p; W.o_totals = g->o_totals.p; W.o_n = g->o_n.p; W.counters = g->counters.p;
    if (sb) {
      W.k1p1 = sb->k1 + 1.0f;  // constants.k1 + 1.0 in f32 (core/src/ranking/bm25.rs:149)
      W.coeff_text = sb->coeff_text; W.max_docs = sb->max_docs;
      if (sb->signals && sb->signals->n_cols) {
        if (sb->signals->max_doc < g->max_doc) SB_FAIL(SB200_EINVAL, "signal table covers %u docs, segment has %u", sb->signals->max_doc, g->max_doc);
        if (!sb->coeffs) SB_FAIL(SB200_EINVAL, "coeffs is NULL");
        SB_TRY(ensure(g->q_coeffs, sb->signals->n_cols));
        SB_CUDA(cudaMemcpyAsync(g->q_coeffs.p, sb->coeffs, sb->signals->n_cols * 8, cudaMemcpyDefault, s));
        W.sig = sb->signals->rows.p; W.n_cols = sb->signals->n_cols; W.coeffs = g->q_coeffs.p;
      }
    }
    if (!sb && mode == SB200_MODE_AND) SB_TRY(launch_topk_warp<0>(W, s));
    else if (sb && sb->max_docs) SB_TRY(launch_topk_warp<2>(W, s));   // k_or3 has no max_docs short circuit
    else if (sb) SB_TRY(launch_or3<2>(W, s));
    else SB_TRY(launch_or3<1>(W, s));
    if (!pl.jobs.empty()) {
      const size_t msm = (size_t)pl.capm * 12;
      static size_t mconf[3] = {0, 0, 0};
      if (sb) { if (msm > 48 * 1024 && mconf[2] < msm) { SB_CUDA(cudaFuncSetAttribute(k_merge_topk<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)msm)); mconf[2] = msm; }
                SB_LAUNCH(k_merge_topk<2>, (unsigned)pl.jobs.size(), 256, msm, s, g->q_jobs.p, k, pl.capm, W.o_docs, W.o_scores, W.o_totals, W.o_n); }
      else { if (msm > 48 * 1024 && mconf[0] < msm) { SB_CUDA(cudaFuncSetAttribute(k_merge_topk<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)msm)); mconf[0] = msm; }
             SB_LAUNCH(k_merge_topk<0>, (unsigned)pl.jobs.size(), 256, msm, s, g->q_jobs.p, k, pl.capm, W.o_docs, W.o_scores, W.o_totals, W.o_n); }
      SB_CHECK_LAUNCH();
    }
  }
  SB_CUDA(cudaEventRecord(g->evk1, s));
  SB_TRY(copy_out_tables(g, nq, k, docs, scores, totals, n_out));
  unsigned long long h[4] = {0, 0, 0, 0};
  SB_CUDA(cudaMemcpyAsync(h, g->counters.p, sizeof(h), cudaMemcpyDeviceToHost, s));
  SB_CUDA(cudaEventRecord(g->ev1, s));
  SB_CUDA(cudaStreamSynchronize(s));
  if (h[2]) SB_FAIL(SB200_EFORMAT, "%llu queries hit the decode watchdog (inconsistent posting data)", h[2]);
  if (stats) {
    float ms = 0; cudaEventElapsedTime(&ms, g->ev0, g->ev1);
    stats->postings_scored = postings; stats->docs_scored = h[0]; stats->blocks_decoded = h[1]; stats->ms = ms; cudaEventElapsedTime(&stats->kernel_ms, g->evk0, g->evk1);
  }
  return SB200_OK;
}

static void pos_view(const sb200_segment* g, PosView& V) {
  V.f32 = (const uint32_t*)g->pos_file.p; V.data_off = g->pos_data_off.p; V.tail_off = g->pos_tail_off.p; V.end_off = g->pos_end_off.p;
  V.count = g->pos_count.p; V.first = g->pos_first.p; V.nblk = g->pos_nblk.p; V.b_off = g->pos_b_off.p; V.b_w = g->pos_b_w.p;
}

// Host planning of phrase rows, as PhraseWeight::phrase_scorer: a term the segment does not hold empties the phrase (its row
// keeps 0 terms); the others are put in Intersection order (stable sort by doc_freq, intersection.rs:69-81) with their shift
// max_offset - offset.
static int phrase_rows(const sb200_segment* g, uint32_t nq, uint32_t nt, const uint32_t* ords_in, const uint32_t* offsets, const uint32_t* slops,
                       std::vector<uint32_t>& terms, std::vector<uint32_t>& shift, std::vector<uint32_t>& nterms, std::vector<uint32_t>& slop) {
  terms.assign((size_t)nq * nt, 0); shift.assign((size_t)nq * nt, 0); nterms.assign(nq, 0); slop.assign(nq, 0);
  for (uint32_t q = 0; q < nq; q++) {
    uint32_t ords[MAXT], offs[MAXT], c = 0;
    bool absent = false;
    for (uint32_t t = 0; t < nt; t++) {
      const uint32_t ord = ords_in[(size_t)q * nt + t];
      if (ord == SB200_NO_TERM) {
        for (uint32_t u = t; u < nt; u++) if (ords_in[(size_t)q * nt + u] != SB200_NO_TERM) SB_FAIL(SB200_EINVAL, "query %u: SB200_NO_TERM pads the end of a row only", q);
        break;
      }
      if (ord == SB200_ABSENT_TERM) absent = true;
      else if (ord >= g->n_terms) SB_FAIL(SB200_EINVAL, "query %u: term ordinal %u >= %u", q, ord, g->n_terms);
      ords[c] = ord; offs[c] = offsets ? offsets[(size_t)q * nt + t] : t; c++;
    }
    if (c < 2) SB_FAIL(SB200_EINVAL, "query %u has %u terms: a phrase has 2..%d", q, c, MAXT);
    slop[q] = slops ? slops[q] : 0u;
    if (absent) continue;
    uint32_t max_off = 0, idx[MAXT];
    for (uint32_t i = 0; i < c; i++) { max_off = std::max(max_off, offs[i]); idx[i] = i; }
    std::stable_sort(idx, idx + c, [&](uint32_t x, uint32_t y) { return g->h_df[ords[x]] < g->h_df[ords[y]]; });
    for (uint32_t i = 0; i < c; i++) { terms[(size_t)q * nt + i] = ords[idx[i]]; shift[(size_t)q * nt + i] = max_off - offs[idx[i]]; }
    nterms[q] = c;
  }
  return SB200_OK;
}

// Candidates (k_phrase_cand<2>) and verification (k_phrase_verify) of planned phrase rows, in groups whose candidate records
// fit a memory budget; scoring == 0 is exists mode.  After a group's verification the matches of row q are at a3_off[q],
// ph_mcnt[q] of them (ph_mkey / ph_mdoc, unordered), and done(g0, g1) consumes rows [g0, g1).  kms accumulates the launches.
typedef std::function<int(uint32_t, uint32_t)> PhraseDone;
static int phrase_match(sb200_segment* g, uint32_t nq, uint32_t nt, const std::vector<uint32_t>& terms, const std::vector<uint32_t>& shift,
                        const std::vector<uint32_t>& nterms, const std::vector<uint32_t>& slop, const std::vector<float>& weight, int scoring,
                        const float* tf_cache256, float& kms, PhraseDone done) {
  cudaStream_t s = g->stream;
  SB_TRY(ensure(g->q_terms, (size_t)nq * nt)); SB_TRY(ensure(g->ph_shift, (size_t)nq * nt)); SB_TRY(ensure(g->q_nterms, nq));
  SB_TRY(ensure(g->ph_slop, nq)); SB_TRY(ensure(g->ph_weight, nq)); SB_TRY(ensure(g->q_weights, (size_t)nq * nt)); SB_TRY(ensure(g->q_cache, 256));
  SB_TRY(ensure(g->counters, 8)); SB_TRY(ensure(g->a3_off, nq)); SB_TRY(ensure(g->a3_cnt, nq)); SB_TRY(ensure(g->ph_mcnt, nq));
  SB_TRY(ensure(g->ph_ovc, 4)); SB_TRY(ensure(g->ph_pre, (size_t)nq + 1));
  SB_CUDA(cudaMemcpyAsync(g->q_terms.p, terms.data(), terms.size() * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->ph_shift.p, shift.data(), shift.size() * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->q_nterms.p, nterms.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->ph_slop.p, slop.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(g->ph_weight.p, weight.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemsetAsync(g->q_weights.p, 0, (size_t)nq * nt * 4, s));
  if (scoring) SB_CUDA(cudaMemcpyAsync(g->q_cache.p, tf_cache256, 256 * 4, cudaMemcpyDefault, s));
  else SB_CUDA(cudaMemsetAsync(g->q_cache.p, 0, 256 * 4, s));
  SB_CUDA(cudaMemsetAsync(g->counters.p, 0, 8 * sizeof(unsigned long long), s));
  SB_CUDA(cudaMemsetAsync(g->a3_cnt.p, 0, (size_t)nq * 4, s));
  SB_CUDA(cudaMemsetAsync(g->ph_mcnt.p, 0, (size_t)nq * 4, s));
  const size_t cand_smem = (size_t)A3_WARPS * nt * 128 * 12;
  static size_t cand_conf = 0;
  if (cand_conf < cand_smem) { SB_CUDA(cudaFuncSetAttribute(k_phrase_cand<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cand_smem)); cand_conf = cand_smem; }
  int n_sm = 132;
  { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev); if (n_sm <= 0) n_sm = 132; }
  // candidate records: doc + nt x (u64 offset, u32 tf) + a match (key, doc) per entry
  uint64_t budget = (uint64_t)2 << 30;
  if (const char* e = getenv("SB200_PHRASE_BUDGET_MB")) { const long mb = atol(e); if (mb > 0) budget = (uint64_t)mb << 20; }
  const uint64_t max_entries = std::max<uint64_t>(budget / (12 + 12 * (uint64_t)nt), 1);
  std::vector<uint64_t> off(nq, 0), pre(nq + 1, 0);
  std::vector<uint32_t> cnt(nq, 0);
  std::vector<AUnit> units;
  auto timed = [&](auto&& launch) -> int {
    SB_CUDA(cudaEventRecord(g->evk0, s));
    SB_TRY(launch());
    SB_CUDA(cudaEventRecord(g->evk1, s));
    SB_CUDA(cudaStreamSynchronize(s));
    float ms = 0.0f; cudaEventElapsedTime(&ms, g->evk0, g->evk1); kms += ms;
    return SB200_OK;
  };
  uint32_t g0 = 0;
  while (g0 < nq) {
    uint64_t entries = 0; uint32_t g1 = g0;
    units.clear();
    while (g1 < nq) {
      const uint32_t dfA = nterms[g1] ? g->h_df[terms[(size_t)g1 * nt]] : 0u;
      if (g1 > g0 && entries + dfA > max_entries) break;
      off[g1] = entries; entries += dfA;
      const uint32_t nblk = (dfA >> 7) + ((dfA & 127u) ? 1u : 0u);
      for (uint32_t b0 = 0; b0 < nblk; b0 += A3_UNIT_BLOCKS) { AUnit u; u.q = g1; u.blk_lo = b0; u.blk_hi = std::min(nblk, b0 + A3_UNIT_BLOCKS); u._pad = 0; units.push_back(u); }
      g1++;
    }
    const uint32_t n_units = (uint32_t)units.size();
    const size_t ne = (size_t)std::max<uint64_t>(entries, 1);
    SB_TRY(ensure(g->ph_cdoc, ne)); SB_TRY(ensure(g->ph_coff, ne * nt)); SB_TRY(ensure(g->ph_ctf, ne * nt));
    SB_TRY(ensure(g->ph_mkey, ne)); SB_TRY(ensure(g->ph_mdoc, ne)); SB_TRY(ensure(g->a3_units, std::max<size_t>(n_units, 1)));
    SB_CUDA(cudaMemcpyAsync(g->a3_off.p + g0, off.data() + g0, (size_t)(g1 - g0) * 8, cudaMemcpyHostToDevice, s));
    if (n_units) {
      SB_CUDA(cudaMemcpyAsync(g->a3_units.p, units.data(), (size_t)n_units * sizeof(AUnit), cudaMemcpyHostToDevice, s));
      PhCandParams C;
      memset(&C, 0, sizeof(C));
      seg_view(g, C.A.S); C.A.a128 = g->a_post.p; C.A.t_aoff = g->t_aoff.p;
      C.A.q_terms = g->q_terms.p; C.A.q_nterms = g->q_nterms.p; C.A.q_weights = g->q_weights.p; C.A.cache = g->q_cache.p; C.A.n_terms_max = nt;
      C.A.units = (const AUnit*)g->a3_units.p; C.A.n_units = n_units;
      C.A.cand_off = g->a3_off.p; C.A.cand_cnt = g->a3_cnt.p; C.A.counters = g->counters.p;
      C.pos_base = g->pos_base.p; C.nt = nt; C.c_doc = g->ph_cdoc.p; C.c_off = g->ph_coff.p; C.c_tf = g->ph_ctf.p;
      SB_TRY(timed([&]() -> int { SB_LAUNCH(k_phrase_cand<2>, div_up(n_units, A3_WARPS), A3_WARPS * 32, cand_smem, s, C); SB_CHECK_LAUNCH(); return SB200_OK; }));
    }
    // candidate counts -> the group's prefix (k_phrase_verify maps a candidate to its query by a binary search in it)
    SB_CUDA(cudaMemcpyAsync(cnt.data() + g0, g->a3_cnt.p + g0, (size_t)(g1 - g0) * 4, cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaStreamSynchronize(s));
    const uint32_t ns = g1 - g0;
    pre[0] = 0;
    for (uint32_t i = 0; i < ns; i++) pre[i + 1] = pre[i] + cnt[g0 + i];
    const uint64_t total = pre[ns];
    if (total) {
      SB_CUDA(cudaMemcpyAsync(g->ph_pre.p, pre.data(), (size_t)(ns + 1) * 8, cudaMemcpyHostToDevice, s));
      SB_TRY(ensure(g->ph_ov, 2 * (size_t)total));
      PhParams V;
      memset(&V, 0, sizeof(V));
      pos_view(g, V.V);
      V.fieldnorm = g->fieldnorm.p; V.cache = g->q_cache.p;
      V.q_terms = g->q_terms.p; V.q_shift = g->ph_shift.p; V.q_nterms = g->q_nterms.p; V.q_slop = g->ph_slop.p; V.q_weight = g->ph_weight.p;
      V.nt = nt; V.scoring = scoring ? 1 : 0;
      V.cand_off = g->a3_off.p; V.cand_pre = g->ph_pre.p; V.slot0 = g0; V.n_slots = ns;
      V.c_doc = g->ph_cdoc.p; V.c_off = g->ph_coff.p; V.c_tf = g->ph_ctf.p;
      V.m_cnt = g->ph_mcnt.p; V.m_key = g->ph_mkey.p; V.m_doc = g->ph_mdoc.p; V.counters = g->counters.p;
      unsigned long long* lists[2] = {(unsigned long long*)g->ph_ov.p, (unsigned long long*)g->ph_ov.p + total};
      V.list = nullptr; V.n = total; V.factor = 1; V.ov_list = lists[0]; V.ov = g->ph_ovc.p; V.scratch_cursor = g->ph_ovc.p + 2;
      SB_CUDA(cudaMemsetAsync(g->ph_ovc.p, 0, 4 * sizeof(unsigned long long), s));
      const unsigned grid = (unsigned)std::min<uint64_t>(div_up(total, PH_WARPS), (uint64_t)n_sm * 16);
      SB_TRY(timed([&]() -> int { SB_LAUNCH(k_phrase_verify, grid, PH_WARPS * 32, 0, s, V); SB_CHECK_LAUNCH(); return SB200_OK; }));
      // candidates whose lists do not fit shared memory, then those whose carrying-slop merge outgrew its buffers
      uint64_t factor = 1;
      for (int pass = 0;; pass++) {
        unsigned long long ov[4] = {0, 0, 0, 0};
        SB_CUDA(cudaMemcpyAsync(ov, g->ph_ovc.p, sizeof(ov), cudaMemcpyDeviceToHost, s));
        SB_CUDA(cudaStreamSynchronize(s));
        if (ov[0] == 0) break;
        if (pass >= 8) SB_FAIL(SB200_ENOMEM, "phrase verification: the carrying-slop buffers of %llu candidates still overflow", ov[0]);
        factor = std::max<uint64_t>(factor * 4, ov[3]);   // 4x, or the merge length the overflowing candidates asked for
        if (factor > 0xFFFFFFFFull) SB_FAIL(SB200_ENOMEM, "phrase verification: carrying-slop buffers beyond 2^32 entries");
        SB_TRY(ensure(g->ph_scratch, (size_t)(ov[1] * (1 + 4ull * factor) + 64)));
        V.list = lists[pass & 1]; V.n = ov[0]; V.ov_list = lists[(pass + 1) & 1];
        V.scratch = g->ph_scratch.p; V.factor = (uint32_t)factor;
        SB_CUDA(cudaMemsetAsync(g->ph_ovc.p, 0, 4 * sizeof(unsigned long long), s));
        const unsigned grid2 = (unsigned)std::min<uint64_t>(div_up(ov[0], PH_WARPS), (uint64_t)n_sm * 16);
        SB_TRY(timed([&]() -> int { SB_LAUNCH(k_phrase_verify, grid2, PH_WARPS * 32, 0, s, V); SB_CHECK_LAUNCH(); return SB200_OK; }));
      }
    }
    SB_TRY(done(g0, g1));
    g0 = g1;
  }
  return SB200_OK;
}

template <int TMAX>
static int launch_wp_signals(const WpParams& W, cudaStream_t s) {
  const size_t sm = wp_cta_smem<TMAX>();
  static bool configured = false;
  if (!configured) { SB_CUDA(cudaFuncSetAttribute(k_wp_signals<TMAX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm)); configured = true; }
  SB_LAUNCH(k_wp_signals<TMAX>, div_up(W.n_units, WQ), WQ * 32, sm, s, W);
  SB_CHECK_LAUNCH();
  return SB200_OK;
}

// Recall webpages (bm25_webpage.cuh) of the caller's documents, after run_multi uploaded the slots (query order kept, text slots
// first) and the optic tables: sort, k_wp_signals, then k_wp_slop over the (document, distance field) pairs that need positions --
// a shared-memory pass and a global-scratch pass for the pairs whose lists do not fit.  sb200_multi_signal_webpages checked wp.b.
static int run_webpages(sb200_segment* g, const MParams& P, const sb200_multi_signal_batch* b, const std::vector<uint8_t>& sf,
                        const std::vector<uint32_t>& ns, const WpCall& wp) {
  const sb200_webpage_batch* wb = wp.b;
  const sb200_webpage_out* out = wp.out;
  cudaStream_t s = g->stream;
  const uint32_t nq = wb->n_queries, ndm = wb->n_docs_max, SM = b->n_slots, NO = b->n_ops;
  const size_t n_out = (size_t)nq * ndm;
  // keys in the caller's order, each query's range and its 32-key chunks
  std::vector<uint32_t> beg(nq + 1, 0), units;
  for (uint32_t q = 0; q < nq; q++) beg[q + 1] = beg[q] + wb->n_docs[q];
  const uint32_t n_keys = beg[nq];
  std::vector<uint64_t> keys(n_keys);
  std::vector<uint32_t> idx(n_keys);
  for (uint32_t q = 0; q < nq; q++) {
    for (uint32_t i = 0; i < wb->n_docs[q]; i++) {
      keys[beg[q] + i] = ((uint64_t)q << 32) | wb->docs[(size_t)q * ndm + i];
      idx[beg[q] + i] = (uint32_t)((size_t)q * ndm + i);
    }
    for (uint32_t c = 0; c < wb->n_docs[q]; c += 32) units.push_back(beg[q] + c);
  }
  // row width of the offset scratch: the distance fields' text slots of a query, at most
  uint32_t nd = 1;
  for (uint32_t q = 0; q < nq; q++) {
    uint32_t c = 0;
    for (uint32_t x = 0; x < ns[q]; x++) { const uint8_t f = sf[(size_t)q * SM + x]; if (f == wb->dist_field[0] || f == wb->dist_field[1]) c++; }
    nd = std::max(nd, c);
  }
  const size_t nk = std::max<size_t>(n_keys, 1);
  SB_TRY(ensure(g->wp_keys, nk)); SB_TRY(ensure(g->wp_keys2, nk)); SB_TRY(ensure(g->wp_idx, nk)); SB_TRY(ensure(g->wp_idx2, nk));
  SB_TRY(ensure(g->wp_beg, nq + 1)); SB_TRY(ensure(g->wp_units, std::max<size_t>(units.size(), 1)));
  SB_TRY(ensure(g->wp_off, nk * nd)); SB_TRY(ensure(g->wp_tf, nk * nd)); SB_TRY(ensure(g->wp_work, 2 * nk)); SB_TRY(ensure(g->wp_ovl, 2 * nk));
  SB_TRY(ensure(g->wp_ovc, 4)); SB_TRY(ensure(g->counters, 8));
  const size_t no = std::max<size_t>(n_out, 1);
  SB_TRY(ensure(g->wp_values, no * NO)); SB_TRY(ensure(g->wp_scores, no * NO)); SB_TRY(ensure(g->wp_boosts, no)); SB_TRY(ensure(g->wp_slop, no * 2));
  float kms = 0.0f;
  auto timed = [&](auto&& launch) -> int {
    SB_CUDA(cudaEventRecord(g->evk0, s));
    SB_TRY(launch());
    SB_CUDA(cudaEventRecord(g->evk1, s));
    SB_CUDA(cudaStreamSynchronize(s));
    float ms = 0.0f; cudaEventElapsedTime(&ms, g->evk0, g->evk1); kms += ms;
    return SB200_OK;
  };
  if (n_out) {   // values of the numeric ops are not written: keep the caller's
    SB_CUDA(cudaMemcpyAsync(g->wp_values.p, out->values, n_out * NO * 8, cudaMemcpyDefault, s));
    SB_CUDA(cudaMemsetAsync(g->wp_scores.p, 0, n_out * NO * 8, s));
    SB_CUDA(cudaMemsetAsync(g->wp_boosts.p, 0, n_out * 8, s));
    SB_CUDA(cudaMemsetAsync(g->wp_slop.p, 0, n_out * 8, s));
  }
  SB_CUDA(cudaMemsetAsync(g->counters.p, 0, 8 * sizeof(unsigned long long), s));
  SB_CUDA(cudaMemsetAsync(g->wp_ovc.p, 0, 4 * sizeof(unsigned long long), s));
  unsigned long long h[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (n_keys) {
    SB_CUDA(cudaMemcpyAsync(g->wp_keys.p, keys.data(), (size_t)n_keys * 8, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(g->wp_idx.p, idx.data(), (size_t)n_keys * 4, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(g->wp_beg.p, beg.data(), (size_t)(nq + 1) * 4, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(g->wp_units.p, units.data(), units.size() * 4, cudaMemcpyHostToDevice, s));
    int qbits = 1; while ((1ull << qbits) < nq) qbits++;
    cub::DoubleBuffer<uint64_t> dk((uint64_t*)g->wp_keys.p, (uint64_t*)g->wp_keys2.p);
    cub::DoubleBuffer<uint32_t> dv(g->wp_idx.p, g->wp_idx2.p);
    size_t need = 0;
    SB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, need, dk, dv, (int64_t)n_keys, 0, 32 + qbits, s));
    SB_TRY(ensure(g->wp_tmp, need + 256));
    SB_TRY(timed([&]() -> int { SB_CUDA(cub::DeviceRadixSort::SortPairs(g->wp_tmp.p, need, dk, dv, (int64_t)n_keys, 0, 32 + qbits, s)); return SB200_OK; }));
    WpParams W;
    memset(&W, 0, sizeof(W));
    W.M = P;
    W.keys = dk.Current(); W.idx = dv.Current(); W.q_beg = g->wp_beg.p; W.units = g->wp_units.p; W.n_units = (uint32_t)units.size();
    for (int f = 0; f < 2; f++) {
      W.dist[f] = wb->dist_field[f];
      W.pos_base[f] = wb->dist_field[f] == SB200_WEBPAGE_NO_FIELD ? nullptr : b->fields[wb->dist_field[f]].seg->pos_base.p;
    }
    W.nd = nd; W.s_off = g->wp_off.p; W.s_tf = g->wp_tf.p;
    W.o_values = g->wp_values.p; W.o_scores = g->wp_scores.p; W.o_boosts = g->wp_boosts.p; W.o_slop = g->wp_slop.p;
    W.work = (unsigned long long*)g->wp_work.p; W.counters = g->counters.p;
    SB_TRY(timed([&]() -> int { if (SM <= 8) return launch_wp_signals<8>(W, s); return launch_wp_signals<16>(W, s); }));
    SB_CUDA(cudaMemcpyAsync(h, g->counters.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaStreamSynchronize(s));
    if (h[1]) SB_FAIL(SB200_EFORMAT, "%llu chunks met inconsistent posting data", h[1]);
    if (h[0]) {
      int n_sm = 132;
      { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev); if (n_sm <= 0) n_sm = 132; }
      WpSlopParams Q;
      memset(&Q, 0, sizeof(Q));
      for (int f = 0; f < 2; f++) {
        Q.dist[f] = wb->dist_field[f];
        if (wb->dist_field[f] != SB200_WEBPAGE_NO_FIELD) pos_view(b->fields[wb->dist_field[f]].seg, Q.V[f]);
      }
      Q.keys = W.keys; Q.idx = W.idx;
      Q.q_slot_field = P.q_slot_field; Q.q_slot_term = P.q_slot_term; Q.q_nslots = P.q_nslots; Q.n_slots_max = SM;
      Q.nd = nd; Q.s_off = g->wp_off.p; Q.s_tf = g->wp_tf.p;
      Q.work = W.work; Q.n = h[0];
      Q.ov_list = (unsigned long long*)g->wp_ovl.p; Q.ov = (unsigned long long*)g->wp_ovc.p; Q.scratch_cursor = Q.ov + 2;
      Q.o_slop = g->wp_slop.p; Q.counters = g->counters.p;
      const unsigned grid = (unsigned)std::min<uint64_t>(div_up(h[0], PH_WARPS), (uint64_t)n_sm * 16);
      SB_TRY(timed([&]() -> int { SB_LAUNCH(k_wp_slop, grid, PH_WARPS * 32, 0, s, Q); SB_CHECK_LAUNCH(); return SB200_OK; }));
      unsigned long long ov[4] = {0, 0, 0, 0};
      SB_CUDA(cudaMemcpyAsync(ov, g->wp_ovc.p, sizeof(ov), cudaMemcpyDeviceToHost, s));
      SB_CUDA(cudaStreamSynchronize(s));
      if (ov[0]) {   // the lists of these pairs do not fit shared memory: one pass over global scratch sized by their total
        SB_TRY(ensure(g->wp_scratch, (size_t)ov[1] + 64));
        SB_CUDA(cudaMemcpyAsync(g->wp_work.p, g->wp_ovl.p, ov[0] * 8, cudaMemcpyDeviceToDevice, s));
        SB_CUDA(cudaMemsetAsync(g->wp_ovc.p, 0, 4 * sizeof(unsigned long long), s));
        Q.work = (const unsigned long long*)g->wp_work.p; Q.n = ov[0]; Q.scratch = g->wp_scratch.p;
        const unsigned grid2 = (unsigned)std::min<uint64_t>(div_up(ov[0], PH_WARPS), (uint64_t)n_sm * 16);
        SB_TRY(timed([&]() -> int { SB_LAUNCH(k_wp_slop, grid2, PH_WARPS * 32, 0, s, Q); SB_CHECK_LAUNCH(); return SB200_OK; }));
      }
      SB_CUDA(cudaMemcpyAsync(h, g->counters.p, sizeof(h), cudaMemcpyDeviceToHost, s));
      SB_CUDA(cudaStreamSynchronize(s));
      if (h[1]) SB_FAIL(SB200_EFORMAT, "%llu documents met inconsistent posting or positions data", h[1]);
    }
  }
  if (n_out) {
    SB_CUDA(cudaMemcpyAsync(out->values, g->wp_values.p, n_out * NO * 8, cudaMemcpyDefault, s));
    SB_CUDA(cudaMemcpyAsync(out->scores, g->wp_scores.p, n_out * NO * 8, cudaMemcpyDefault, s));
    SB_CUDA(cudaMemcpyAsync(out->boosts, g->wp_boosts.p, n_out * 8, cudaMemcpyDefault, s));
    SB_CUDA(cudaMemcpyAsync(out->min_slop, g->wp_slop.p, n_out * 8, cudaMemcpyDefault, s));
  }
  SB_CUDA(cudaEventRecord(g->ev1, s));
  SB_CUDA(cudaStreamSynchronize(s));
  if (wp.stats) {
    float ms = 0; cudaEventElapsedTime(&ms, g->ev0, g->ev1);
    wp.stats->docs = n_keys; wp.stats->docs_with_positions = h[2]; wp.stats->positions_decoded = h[3]; wp.stats->position_bytes = h[4];
    wp.stats->ms = ms; wp.stats->kernel_ms = kms;
  }
  return SB200_OK;
}

// Phrase batch (bm25_phrase.cuh): phrase_rows, phrase_match, then k_and3_select takes every group's top k.
static int run_phrase(sb200_segment* g, const sb200_phrase_batch* b, uint32_t* docs, float* scores, uint32_t* n_out, sb200_phrase_stats* stats) {
  NvtxRange nvtx("sb200 phrase top-k batch");
  cudaStream_t s = g->stream;
  if (!b || !b->term_ords || !docs || !scores || !n_out) SB_FAIL(SB200_EINVAL, "NULL argument");
  if (b->scoring && (!b->weights || !b->tf_cache256)) SB_FAIL(SB200_EINVAL, "scoring needs weights and tf_cache256");
  if (g->record != SB200_RECORD_FREQS_POSITIONS) SB_FAIL(SB200_EINVAL, "phrase query on a field without positions (record option %d)", g->record);
  if (!g->has_pos) SB_FAIL(SB200_EINVAL, "phrase query: no positions attached to the segment (sb200_segment_attach_positions)");
  const uint32_t nq = b->n_queries, nt = b->n_terms, k = b->k;
  if (nt < 2 || nt > MAXT) SB_FAIL(SB200_ERANGE, "n_terms %u outside [2,%d]", nt, MAXT);
  if (k == 0 || k > SB200_MAX_K) SB_FAIL(SB200_ERANGE, "k %u outside [1,%d]", k, SB200_MAX_K);
  if (stats) memset(stats, 0, sizeof(*stats));
  if (nq == 0) return SB200_OK;
  std::vector<uint32_t> terms, shift, nterms, slop;
  SB_TRY(phrase_rows(g, nq, nt, b->term_ords, b->offsets, b->slop, terms, shift, nterms, slop));
  std::vector<float> weight(nq, 0.0f);
  for (uint32_t q = 0; q < nq; q++) weight[q] = b->scoring ? b->weights[q] : 0.0f;
  SB_TRY(ensure(g->o_docs, (size_t)nq * k)); SB_TRY(ensure(g->o_scores, (size_t)nq * k)); SB_TRY(ensure(g->o_n, nq));
  SB_CUDA(cudaEventRecord(g->ev0, s));
  static size_t sel_conf = 0;
  const size_t sel_smem = (size_t)A3_SEL_CAP * 8;
  if (sel_conf < sel_smem) { SB_CUDA(cudaFuncSetAttribute(k_and3_select, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sel_smem)); sel_conf = sel_smem; }
  float kms = 0.0f;
  SB_TRY(phrase_match(g, nq, nt, terms, shift, nterms, slop, weight, b->scoring, b->tf_cache256, kms, [&](uint32_t g0, uint32_t g1) -> int {
    SB_CUDA(cudaEventRecord(g->evk0, s));
    SB_LAUNCH(k_and3_select, g1 - g0, 256, sel_smem, s, g->a3_off.p, g->ph_mcnt.p, g->ph_mkey.p, g->ph_mdoc.p, (const uint32_t*)nullptr, g0, k,
              g->o_docs.p, g->o_scores.p, g->o_n.p);
    SB_CHECK_LAUNCH();
    SB_CUDA(cudaEventRecord(g->evk1, s));
    SB_CUDA(cudaStreamSynchronize(s));
    float ms = 0.0f; cudaEventElapsedTime(&ms, g->evk0, g->evk1); kms += ms;
    return SB200_OK; }));
  SB_TRY(copy_out_tables(g, nq, k, docs, scores, nullptr, n_out));
  unsigned long long h[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  SB_CUDA(cudaMemcpyAsync(h, g->counters.p, sizeof(h), cudaMemcpyDeviceToHost, s));
  SB_CUDA(cudaEventRecord(g->ev1, s));
  SB_CUDA(cudaStreamSynchronize(s));
  if (h[2]) SB_FAIL(SB200_EFORMAT, "%llu phrase work items met inconsistent posting / position data", h[2]);
  if (h[5]) SB_FAIL(SB200_ENOMEM, "phrase verification: %llu candidates need carrying-slop buffers beyond 2^32 entries", h[5]);
  if (stats) {
    stats->candidates = h[0]; stats->matches = h[1]; stats->positions_decoded = h[3]; stats->position_bytes = h[4];
    cudaEventElapsedTime(&stats->ms, g->ev0, g->ev1); stats->kernel_ms = kms;
  }
  return SB200_OK;
}


// Plan docset stage (bm25_plan.cuh).  The host validates every program, picks each query's cover (BooleanWeight's docset is a
// subset of it) and splits the batch into groups whose cover fits a memory budget; per group the device decodes the cover,
// sorts it, runs the programs on it and compacts the survivors, and `emit` receives them: keys (query in group << 32 | doc),
// ascending, and q_beg, each query's range in them (device and host copies).
static int run_plan(const sb200_recall_plan_batch* pb, PlanEmit emit, sb200_plan_stats* stats) {
  NvtxRange nvtx("sb200 recall plan docsets");
  if (!pb || !pb->segments || pb->n_segments == 0 || !pb->node_off) SB_FAIL(SB200_EINVAL, "NULL argument");
  const uint32_t nq = pb->n_queries, NS = pb->n_segments;
  sb200_segment* g = pb->segments[0];
  if (!g) SB_FAIL(SB200_EINVAL, "plan segment 0 is NULL");
  for (uint32_t i = 0; i < NS; i++) {
    const sb200_segment* x = pb->segments[i];
    if (!x || x->device != g->device || x->max_doc != g->max_doc) SB_FAIL(SB200_EINVAL, "plan segment %u: NULL, or another max_doc / device than segment 0", i);
  }
  if (nq && pb->node_off[nq] > pb->node_off[0] && !pb->nodes) SB_FAIL(SB200_EINVAL, "NULL nodes");
  const auto t0 = std::chrono::steady_clock::now();
  SB_CUDA(cudaSetDevice(g->device));
  cudaStream_t s = g->stream;
  // ---- phrase leaves: every distinct (segment, row) is planned once (phrase_rows); its matching documents come later
  const uint32_t PT = pb->phrase_terms;
  std::vector<std::vector<uint32_t>> seg_rows(NS);          // per segment: the phrase rows its PHRASE nodes use
  std::vector<uint32_t> ph_index;                           // per node of the batch: the distinct phrase of a PHRASE node
  std::vector<uint64_t> ph_key;                             // per distinct phrase: segment << 32 | row
  {
    const uint32_t nn = nq ? pb->node_off[nq] : 0u;
    ph_index.assign(nn, 0);
    for (uint32_t x = 0; x < nn; x++) {
      const sb200_plan_node& N = pb->nodes[x];
      if (N.kind != SB200_PLAN_PHRASE) continue;
      if (N.segment >= NS) SB_FAIL(SB200_EINVAL, "node %u: segment %u >= %u", x, N.segment, NS);
      if (N.arg >= pb->n_phrases || !pb->phrase_ords) SB_FAIL(SB200_EINVAL, "node %u: phrase row %u >= %u", x, N.arg, pb->n_phrases);
      const sb200_segment* sg = pb->segments[N.segment];
      if (sg->record != SB200_RECORD_FREQS_POSITIONS || !sg->has_pos) SB_FAIL(SB200_EINVAL, "node %u: phrase leaf on plan segment %u, which has no positions", x, N.segment);
      ph_key.push_back(((uint64_t)N.segment << 32) | N.arg);
    }
    std::sort(ph_key.begin(), ph_key.end()); ph_key.erase(std::unique(ph_key.begin(), ph_key.end()), ph_key.end());
    for (uint32_t x = 0; x < nn; x++) if (pb->nodes[x].kind == SB200_PLAN_PHRASE)
      ph_index[x] = (uint32_t)(std::lower_bound(ph_key.begin(), ph_key.end(), ((uint64_t)pb->nodes[x].segment << 32) | pb->nodes[x].arg) - ph_key.begin());
    if (!ph_key.empty() && (PT < 2 || PT > (uint32_t)MAXT)) SB_FAIL(SB200_ERANGE, "phrase_terms %u outside [2,%d]", PT, MAXT);
    for (uint64_t kk : ph_key) seg_rows[kk >> 32].push_back((uint32_t)kk);
  }
  // per segment with phrases: the planned rows (terms in Intersection order; nterms 0 = a term is absent, the phrase is empty)
  std::vector<std::vector<uint32_t>> pr_terms(NS), pr_shift(NS), pr_nterms(NS), pr_slop(NS);
  for (uint32_t si = 0; si < NS; si++) {
    const std::vector<uint32_t>& rows = seg_rows[si];
    if (rows.empty()) continue;
    std::vector<uint32_t> ords(rows.size() * PT), offs(rows.size() * PT), sl(rows.size());
    for (size_t i = 0; i < rows.size(); i++) {
      for (uint32_t t = 0; t < PT; t++) {
        ords[i * PT + t] = pb->phrase_ords[(size_t)rows[i] * PT + t];
        offs[i * PT + t] = pb->phrase_offsets ? pb->phrase_offsets[(size_t)rows[i] * PT + t] : t;
      }
      sl[i] = pb->phrase_slop ? pb->phrase_slop[rows[i]] : 0u;
    }
    SB_TRY(phrase_rows(pb->segments[si], (uint32_t)rows.size(), PT, ords.data(), offs.data(), sl.data(), pr_terms[si], pr_shift[si], pr_nterms[si], pr_slop[si]));
  }
  auto ph_plan = [&](uint32_t i, uint32_t& si, uint32_t& r) {   // distinct phrase -> (segment, index among its rows)
    si = (uint32_t)(ph_key[i] >> 32);
    r = (uint32_t)(std::lower_bound(seg_rows[si].begin(), seg_rows[si].end(), (uint32_t)ph_key[i]) - seg_rows[si].begin());
  };
  // ---- programs and covers
  struct Cov { uint64_t cost = 0; std::vector<uint64_t> leaves; };   // leaves: segment << 32 | ordinal
  std::vector<std::vector<uint64_t>> cover(nq);
  std::vector<uint64_t> cost(nq, 0);
  for (uint32_t q = 0; q < nq; q++) {
    const uint32_t n0 = pb->node_off[q], n1 = pb->node_off[q + 1];
    if (n1 < n0 || n1 - n0 == 0 || n1 - n0 > SB200_PLAN_MAX_NODES) SB_FAIL(SB200_EINVAL, "query %u: %d nodes (1..%d)", q, (int)(n1 - n0), SB200_PLAN_MAX_NODES);
    std::vector<Cov> st;
    std::vector<uint8_t> occ;
    for (uint32_t x = n0; x < n1; x++) {
      const sb200_plan_node& N = pb->nodes[x];
      if (N.occur > SB200_PLAN_MUST_NOT) SB_FAIL(SB200_EINVAL, "query %u node %u: occur %u", q, x - n0, (unsigned)N.occur);
      Cov c;
      if (N.kind == SB200_PLAN_TERM) {
        if (N.segment >= NS) SB_FAIL(SB200_EINVAL, "query %u node %u: segment %u >= %u", q, x - n0, N.segment, NS);
        if (N.arg != SB200_ABSENT_TERM) {
          const sb200_segment* sg = pb->segments[N.segment];
          if (N.arg >= sg->n_terms) SB_FAIL(SB200_EINVAL, "query %u node %u: term ordinal %u >= %u", q, x - n0, N.arg, sg->n_terms);
          c.cost = sg->h_df[N.arg]; c.leaves.push_back(((uint64_t)N.segment << 32) | N.arg);
        }
      } else if (N.kind == SB200_PLAN_PHRASE) {   // cover: the postings of the phrase's rarest term
        uint32_t si, r;
        ph_plan(ph_index[x], si, r);
        if (pr_nterms[si][r]) {
          const uint32_t ord = pr_terms[si][(size_t)r * PT];
          c.cost = pb->segments[si]->h_df[ord]; c.leaves.push_back(((uint64_t)si << 32) | ord);
        }
      } else if (N.kind == SB200_PLAN_BOOL) {
        const uint32_t nc = N.n_children;
        if (nc > st.size()) SB_FAIL(SB200_EINVAL, "query %u node %u: %u children, %zu values on the stack", q, x - n0, nc, st.size());
        const size_t b = st.size() - nc;
        bool has_must = false;
        for (size_t i = b; i < st.size(); i++) has_must |= occ[i] == SB200_PLAN_MUST;
        if (nc == 1 && occ[b] != SB200_PLAN_MUST_NOT) c = st[b];
        else if (nc > 1 && has_must) {   // the cheapest Must clause
          size_t best = SIZE_MAX;
          for (size_t i = b; i < st.size(); i++) if (occ[i] == SB200_PLAN_MUST && (best == SIZE_MAX || st[i].cost < st[best].cost)) best = i;
          c = st[best];
        } else if (nc > 1) {             // the union of the Should clauses
          for (size_t i = b; i < st.size(); i++) if (occ[i] == SB200_PLAN_SHOULD) { c.cost += st[i].cost; c.leaves.insert(c.leaves.end(), st[i].leaves.begin(), st[i].leaves.end()); }
        }
        st.resize(b); occ.resize(b);
      } else if (N.kind != SB200_PLAN_EMPTY) {
        SB_FAIL(SB200_EINVAL, "query %u node %u: kind %u", q, x - n0, (unsigned)N.kind);
      }
      st.push_back(std::move(c)); occ.push_back(N.occur);
    }
    if (st.size() != 1) SB_FAIL(SB200_EINVAL, "query %u: the program leaves %zu values (1 expected)", q, st.size());
    std::vector<uint64_t>& L = st[0].leaves;
    std::sort(L.begin(), L.end()); L.erase(std::unique(L.begin(), L.end()), L.end());
    for (uint64_t l : L) cost[q] += pb->segments[l >> 32]->h_df[(uint32_t)l];
    cover[q] = std::move(L);
  }
  // ---- the matching documents of every distinct phrase (exists mode), ascending, concatenated in ph_key order
  float kms = 0.0f;
  std::vector<uint32_t> ph_off(ph_key.size() + 1, 0), ph_docs;
  {
    std::vector<std::vector<uint32_t>> lists(ph_key.size());
    for (uint32_t si = 0; si < NS; si++) {
      const uint32_t nr = (uint32_t)seg_rows[si].size();
      if (!nr) continue;
      sb200_segment* sg = pb->segments[si];
      const uint32_t base = (uint32_t)(std::lower_bound(ph_key.begin(), ph_key.end(), (uint64_t)si << 32) - ph_key.begin());
      std::vector<float> w(nr, 0.0f);
      std::vector<uint32_t> mc; std::vector<uint64_t> mo;
      SB_TRY(phrase_match(sg, nr, PT, pr_terms[si], pr_shift[si], pr_nterms[si], pr_slop[si], w, 0, nullptr, kms, [&](uint32_t a0, uint32_t a1) -> int {
        mc.resize(a1 - a0); mo.resize(a1 - a0);
        SB_CUDA(cudaMemcpyAsync(mc.data(), sg->ph_mcnt.p + a0, (size_t)(a1 - a0) * 4, cudaMemcpyDeviceToHost, sg->stream));
        SB_CUDA(cudaMemcpyAsync(mo.data(), sg->a3_off.p + a0, (size_t)(a1 - a0) * 8, cudaMemcpyDeviceToHost, sg->stream));
        SB_CUDA(cudaStreamSynchronize(sg->stream));
        for (uint32_t i = 0; i < a1 - a0; i++) {
          std::vector<uint32_t>& L = lists[base + a0 + i];
          L.resize(mc[i]);
          if (mc[i]) SB_CUDA(cudaMemcpy(L.data(), sg->ph_mdoc.p + mo[i], (size_t)mc[i] * 4, cudaMemcpyDeviceToHost));
          std::sort(L.begin(), L.end());
        }
        return SB200_OK; }));
      unsigned long long h[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      SB_CUDA(cudaMemcpyAsync(h, sg->counters.p, sizeof(h), cudaMemcpyDeviceToHost, sg->stream));
      SB_CUDA(cudaStreamSynchronize(sg->stream));
      if (h[2]) SB_FAIL(SB200_EFORMAT, "%llu phrase work items met inconsistent posting / position data", h[2]);
      if (h[5]) SB_FAIL(SB200_ENOMEM, "phrase verification: %llu candidates need carrying-slop buffers beyond 2^32 entries", h[5]);
    }
    for (size_t i = 0; i < lists.size(); i++) {
      if ((uint64_t)ph_docs.size() + lists[i].size() > 0xFFFFFFFFull) SB_FAIL(SB200_ERANGE, "phrase leaves match more than 2^32 documents in all");
      ph_docs.insert(ph_docs.end(), lists[i].begin(), lists[i].end());
      ph_off[i + 1] = (uint32_t)ph_docs.size();
    }
  }
  std::vector<sb200_plan_node> hn(pb->nodes, pb->nodes + (nq ? pb->node_off[nq] : 0u));   // PHRASE args -> distinct phrase
  for (size_t x = 0; x < hn.size(); x++) if (hn[x].kind == SB200_PLAN_PHRASE) hn[x].arg = ph_index[x];
  SB_TRY(ensure(g->pl_ph_off, ph_off.size())); SB_TRY(ensure(g->pl_ph_docs, std::max<size_t>(ph_docs.size(), 1)));
  SB_CUDA(cudaMemcpyAsync(g->pl_ph_off.p, ph_off.data(), ph_off.size() * 4, cudaMemcpyHostToDevice, s));
  if (!ph_docs.empty()) SB_CUDA(cudaMemcpyAsync(g->pl_ph_docs.p, ph_docs.data(), ph_docs.size() * 4, cudaMemcpyHostToDevice, s));
  std::vector<PSeg> hs(NS);
  for (uint32_t i = 0; i < NS; i++) {
    memset(&hs[i], 0, sizeof(PSeg));
    const sb200_segment* x = pb->segments[i];
    seg_view(x, hs[i].S); hs[i].a128 = x->a_post.p; hs[i].t_aoff = x->t_aoff.p; hs[i].n_terms = x->n_terms;
  }
  SB_TRY(ensure(g->pl_segs, NS * sizeof(PSeg))); SB_TRY(ensure(g->counters, 4));
  SB_CUDA(cudaMemcpyAsync(g->pl_segs.p, hs.data(), NS * sizeof(PSeg), cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemsetAsync(g->counters.p, 0, 4 * sizeof(unsigned long long), s));
  // candidate keys twice (sort), a flag, the compacted keys: ~32 B per candidate
  uint64_t budget = (uint64_t)2 << 30;
  if (const char* e = getenv("SB200_PLAN_BUDGET_MB")) { const long mb = atol(e); if (mb > 0) budget = (uint64_t)mb << 20; }
  const uint64_t max_entries = std::max<uint64_t>(budget / 32, 1);
  uint64_t n_cover = 0, n_docs = 0;
  uint32_t n_groups = 0;
  auto timed = [&](auto&& launch) -> int {
    SB_CUDA(cudaEventRecord(g->evk0, s));
    SB_TRY(launch());
    SB_CUDA(cudaEventRecord(g->evk1, s));
    SB_CUDA(cudaStreamSynchronize(s));
    float ms = 0.0f; cudaEventElapsedTime(&ms, g->evk0, g->evk1); kms += ms;
    return SB200_OK;
  };
  std::vector<PCover> units;
  std::vector<uint32_t> chunks, noff;
  std::vector<uint64_t> beg;
  uint32_t g0 = 0;
  while (g0 < nq) {
    uint64_t E = 0; uint32_t g1 = g0;
    while (g1 < nq && (g1 == g0 || E + cost[g1] <= max_entries)) E += cost[g1++];
    const uint32_t n = g1 - g0;
    units.clear(); chunks.clear(); noff.assign(n + 1, 0); beg.assign(n + 1, 0);
    uint64_t at = 0;
    for (uint32_t i = 0; i < n; i++) {
      beg[i] = at;
      for (uint64_t l : cover[g0 + i]) {
        const uint32_t sg = (uint32_t)(l >> 32), ord = (uint32_t)l, df = pb->segments[sg]->h_df[ord];
        const uint32_t nblk = (df >> 7) + ((df & 127u) ? 1u : 0u);
        for (uint32_t b = 0; b < nblk; b++) { PCover c; c.q = i; c.seg = sg; c.ord = ord; c.blk = b; c.out = at + (uint64_t)b * 128; units.push_back(c); }
        at += df;
      }
      for (uint64_t c = beg[i]; c < at; c += 32) chunks.push_back((uint32_t)c);
      noff[i + 1] = pb->node_off[g0 + i + 1] - pb->node_off[g0];
    }
    beg[n] = at;
    const size_t ne = std::max<uint64_t>(E, 1), nn = noff[n];
    SB_TRY(ensure(g->pl_keys, ne)); SB_TRY(ensure(g->pl_keys2, ne)); SB_TRY(ensure(g->pl_keep, ne)); SB_TRY(ensure(g->pl_beg, n + 1));
    SB_TRY(ensure(g->pl_cover, std::max<size_t>(units.size(), 1) * sizeof(PCover))); SB_TRY(ensure(g->pl_units, std::max<size_t>(chunks.size(), 1)));
    SB_TRY(ensure(g->pl_nodes, nn * sizeof(sb200_plan_node))); SB_TRY(ensure(g->pl_off, n + 1)); SB_TRY(ensure(g->pl_cnt, 1));
    SB_CUDA(cudaMemcpyAsync(g->pl_nodes.p, hn.data() + pb->node_off[g0] - pb->node_off[0], nn * sizeof(sb200_plan_node), cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(g->pl_off.p, noff.data(), (size_t)(n + 1) * 4, cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemcpyAsync(g->pl_beg.p, beg.data(), (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, s));
    if (!units.empty()) SB_CUDA(cudaMemcpyAsync(g->pl_cover.p, units.data(), units.size() * sizeof(PCover), cudaMemcpyHostToDevice, s));
    if (!chunks.empty()) SB_CUDA(cudaMemcpyAsync(g->pl_units.p, chunks.data(), chunks.size() * 4, cudaMemcpyHostToDevice, s));
    PlanParams P;
    memset(&P, 0, sizeof(P));
    P.segs = (const PSeg*)g->pl_segs.p; P.nodes = (const sb200_plan_node*)g->pl_nodes.p; P.node_off = g->pl_off.p;
    P.cover = (const PCover*)g->pl_cover.p; P.n_cover = (uint32_t)units.size();
    P.ph_off = g->pl_ph_off.p; P.ph_docs = g->pl_ph_docs.p;
    P.q_beg = g->pl_beg.p; P.units = g->pl_units.p; P.n_units = (uint32_t)chunks.size(); P.keep = g->pl_keep.p; P.counters = g->counters.p;
    uint64_t n_keep = 0;
    if (E) {
      P.keys = g->pl_keys.p; P.n_keys = E;
      SB_TRY(timed([&]() -> int { SB_LAUNCH(k_plan_cover, div_up(units.size(), PL_WARPS), PL_WARPS * 32, 0, s, P); SB_CHECK_LAUNCH(); return SB200_OK; }));
      int qbits = 1; while ((1u << qbits) < n) qbits++;
      cub::DoubleBuffer<uint64_t> dk(g->pl_keys.p, g->pl_keys2.p);
      size_t need = 0;
      SB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, need, dk, (int64_t)E, 0, 32 + qbits, s));
      SB_TRY(ensure(g->pl_tmp, need + 256));
      SB_TRY(timed([&]() -> int { SB_CUDA(cub::DeviceRadixSort::SortKeys(g->pl_tmp.p, need, dk, (int64_t)E, 0, 32 + qbits, s)); return SB200_OK; }));
      P.keys = dk.Current();
      uint64_t* out = dk.Alternate();
      SB_TRY(timed([&]() -> int { SB_LAUNCH(k_plan_eval, div_up(chunks.size(), PL_WARPS), PL_WARPS * 32, 0, s, P); SB_CHECK_LAUNCH(); return SB200_OK; }));
      need = 0;
      SB_CUDA(cub::DeviceSelect::Flagged(nullptr, need, dk.Current(), g->pl_keep.p, out, g->pl_cnt.p, (int64_t)E, s));
      SB_TRY(ensure(g->pl_tmp, need + 256));
      SB_TRY(timed([&]() -> int { SB_CUDA(cub::DeviceSelect::Flagged(g->pl_tmp.p, need, dk.Current(), g->pl_keep.p, out, g->pl_cnt.p, (int64_t)E, s)); return SB200_OK; }));
      SB_CUDA(cudaMemcpyAsync(&n_keep, g->pl_cnt.p, 8, cudaMemcpyDeviceToHost, s));
      SB_CUDA(cudaStreamSynchronize(s));
      SB_TRY(timed([&]() -> int { SB_LAUNCH(k_plan_bounds, div_up(n + 1, 256), 256, 0, s, out, n_keep, n, g->pl_beg.p); SB_CHECK_LAUNCH(); return SB200_OK; }));
      SB_CUDA(cudaMemcpyAsync(beg.data(), g->pl_beg.p, (size_t)(n + 1) * 8, cudaMemcpyDeviceToHost, s));
      unsigned long long h[4] = {0, 0, 0, 0};
      SB_CUDA(cudaMemcpyAsync(h, g->counters.p, sizeof(h), cudaMemcpyDeviceToHost, s));
      SB_CUDA(cudaStreamSynchronize(s));
      if (h[2]) SB_FAIL(SB200_EFORMAT, "%llu plan work items met inconsistent posting data", h[2]);
      P.keys = out;
    } else {
      P.keys = g->pl_keys.p;
    }
    n_cover += E; n_docs += n_keep; n_groups++;
    SB_CUDA(cudaStreamSynchronize(s));   // emit may work on another stream: every upload and launch of the group is complete
    SB_TRY(emit(g0, g1, P.keys, g->pl_beg.p, beg));
    g0 = g1;
  }
  if (stats) {
    stats->cover = n_cover; stats->docs = n_docs; stats->groups = n_groups; stats->_pad = 0;
    stats->ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count(); stats->kernel_ms = kms;
  }
  return SB200_OK;
}


// A new, zeroed docset over the segment's documents
static int docset_new(const sb200_segment* g, sb200_docset** out) {
  sb200_docset* d = new (std::nothrow) sb200_docset;
  if (!d) SB_FAIL(SB200_ENOMEM, "docset: host allocation failed");
  d->device = g->device; d->max_doc = g->max_doc;
  const size_t nw = std::max<size_t>(((size_t)g->max_doc + 31) / 32, 1);
  int rc = d->bits.alloc(nw);
  if (rc == SB200_OK && cudaMemsetAsync(d->bits.p, 0, nw * 4, g->stream) != cudaSuccess) { set_error("docset: memset failed"); rc = SB200_ECUDA; }
  if (rc != SB200_OK) { delete d; return rc; }
  *out = d;
  return SB200_OK;
}

// Pattern batch (bm25_pattern.cuh).  Host planning is PatternWeight::pattern_scorer's branch choice; positional patterns go
// through k_phrase_cand (terms in Intersection order: stable sort by doc_freq) and k_pattern_verify in groups whose candidate
// records fit a memory budget, like run_phrase.
static int run_patterns(sb200_segment* g, const sb200_pattern_batch* b, sb200_docset** out, sb200_pattern_stats* stats) {
  NvtxRange nvtx("sb200 pattern docsets");
  cudaStream_t s = g->stream;
  if (!b || !out || (b->n_patterns && b->n_parts && !b->parts)) SB_FAIL(SB200_EINVAL, "NULL argument");
  const uint32_t np_ = b->n_patterns, NP = b->n_parts, NT = b->n_terms;
  if (NT > (uint32_t)MAXT) SB_FAIL(SB200_ERANGE, "n_terms %u above %d", NT, MAXT);
  if (NT && !b->term_ords) SB_FAIL(SB200_EINVAL, "NULL term_ords");
  if (stats) memset(stats, 0, sizeof(*stats));
  enum { EMPTY, ALL, EMPTY_FIELD, POSTINGS, NORMAL };
  std::vector<int> kind(np_, EMPTY);
  std::vector<uint32_t> nparts(np_, 0), nterms(np_, 0);
  for (uint32_t p = 0; p < np_; p++) {
    uint32_t n = 0, t = 0; bool wild = false, anchor = false, absent = false;
    for (uint32_t i = 0; i < NP; i++) {
      const uint8_t x = b->parts[(size_t)p * NP + i];
      if (x == SB200_PART_PAD) {
        for (uint32_t j = i; j < NP; j++) if (b->parts[(size_t)p * NP + j] != SB200_PART_PAD) SB_FAIL(SB200_EINVAL, "pattern %u: SB200_PART_PAD pads the end of a row only", p);
        break;
      }
      if (x > SB200_PART_ANCHOR) SB_FAIL(SB200_EINVAL, "pattern %u part %u: kind %u", p, i, (unsigned)x);
      if (x == SB200_PART_TERM) {
        if (t >= (uint32_t)MAXT) SB_FAIL(SB200_ERANGE, "pattern %u has more than %d terms", p, MAXT);
        if (t >= NT) SB_FAIL(SB200_EINVAL, "pattern %u has more TERM parts than the row width n_terms %u", p, NT);
        const uint32_t ord = b->term_ords[(size_t)p * NT + t];
        if (ord == SB200_ABSENT_TERM) absent = true;
        else if (ord >= g->n_terms) SB_FAIL(SB200_EINVAL, "pattern %u: term ordinal %u >= %u", p, ord, g->n_terms);
        t++;
      }
      wild |= x == SB200_PART_WILDCARD; anchor |= x == SB200_PART_ANCHOR;
      n++;
    }
    nparts[p] = n; nterms[p] = t;
    if (n == 0) kind[p] = EMPTY;
    else if (t == 0 && wild) kind[p] = ALL;
    else if (t == 0) kind[p] = EMPTY_FIELD;
    else if (absent) kind[p] = EMPTY;
    else if (t == 1 && n == 1) kind[p] = POSTINGS;
    else kind[p] = NORMAL;
    if ((kind[p] == EMPTY_FIELD || (kind[p] == NORMAL && anchor)) && !g->has_tok)
      SB_FAIL(SB200_EINVAL, "pattern %u needs the field's token counts (sb200_segment_attach_token_counts)", p);
    if (kind[p] == NORMAL && (g->record != SB200_RECORD_FREQS_POSITIONS || !g->has_pos))
      SB_FAIL(SB200_EINVAL, "pattern %u needs positions (record option 2 and sb200_segment_attach_positions)", p);
  }
  for (uint32_t p = 0; p < np_; p++) out[p] = nullptr;
  // every docset is created first; on an error the ones made so far are destroyed
  auto fail_cleanup = [&](int rc) { for (uint32_t p = 0; p < np_; p++) { delete out[p]; out[p] = nullptr; } return rc; };
  for (uint32_t p = 0; p < np_; p++) { const int rc = docset_new(g, &out[p]); if (rc != SB200_OK) return fail_cleanup(rc); }
  if (np_ == 0) return SB200_OK;
  int rc = [&]() -> int {
    const uint32_t nw = (g->max_doc + 31) / 32;
    float kms = 0.0f;
    auto timed = [&](auto&& launch) -> int {
      SB_CUDA(cudaEventRecord(g->evk0, s));
      SB_TRY(launch());
      SB_CUDA(cudaEventRecord(g->evk1, s));
      SB_CUDA(cudaStreamSynchronize(s));
      float ms = 0.0f; cudaEventElapsedTime(&ms, g->evk0, g->evk1); kms += ms;
      return SB200_OK;
    };
    SB_CUDA(cudaEventRecord(g->ev0, s));
    SB_TRY(ensure(g->counters, 8));
    SB_CUDA(cudaMemsetAsync(g->counters.p, 0, 8 * sizeof(unsigned long long), s));
    // word kernels
    for (uint32_t p = 0; p < np_; p++) {
      if (kind[p] == ALL) SB_TRY(timed([&]() -> int { SB_LAUNCH(k_docset_all, div_up(nw, 256), 256, 0, s, out[p]->bits.p, g->max_doc); SB_CHECK_LAUNCH(); return SB200_OK; }));
      if (kind[p] == EMPTY_FIELD) SB_TRY(timed([&]() -> int { SB_LAUNCH(k_docset_empty_field, div_up(nw, 256), 256, 0, s, g->tok_count.p, out[p]->bits.p, g->max_doc); SB_CHECK_LAUNCH(); return SB200_OK; }));
    }
    // one-term shortcuts: every posting, one launch for all of them
    std::vector<uint32_t> pq;   // query slot -> pattern
    for (uint32_t p = 0; p < np_; p++) if (kind[p] == POSTINGS) pq.push_back(p);
    SB_TRY(ensure(g->pt_bits, std::max<size_t>(np_, 1)));
    SB_TRY(ensure(g->q_weights, std::max<size_t>((size_t)np_ * std::max<uint32_t>(NT, 1), 1)));
    SB_CUDA(cudaMemsetAsync(g->q_weights.p, 0, std::max<size_t>((size_t)np_ * std::max<uint32_t>(NT, 1), 1) * 4, s));
    std::vector<uint64_t> bp(np_);
    if (!pq.empty()) {
      const uint32_t n1 = (uint32_t)pq.size();
      std::vector<uint32_t> terms(n1), ones(n1, 1);
      std::vector<AUnit> units;
      for (uint32_t i = 0; i < n1; i++) {
        const uint32_t p = pq[i];
        terms[i] = b->term_ords[(size_t)p * NT];
        bp[i] = (uint64_t)(uintptr_t)out[p]->bits.p;
        const uint32_t df = g->h_df[terms[i]], nblk = (df >> 7) + ((df & 127u) ? 1u : 0u);
        for (uint32_t b0 = 0; b0 < nblk; b0 += A3_UNIT_BLOCKS) { AUnit u; u.q = i; u.blk_lo = b0; u.blk_hi = std::min(nblk, b0 + A3_UNIT_BLOCKS); u._pad = 0; units.push_back(u); }
      }
      SB_TRY(ensure(g->q_terms, n1)); SB_TRY(ensure(g->q_nterms, n1)); SB_TRY(ensure(g->a3_units, std::max<size_t>(units.size(), 1)));
      SB_CUDA(cudaMemcpyAsync(g->q_terms.p, terms.data(), (size_t)n1 * 4, cudaMemcpyHostToDevice, s));
      SB_CUDA(cudaMemcpyAsync(g->q_nterms.p, ones.data(), (size_t)n1 * 4, cudaMemcpyHostToDevice, s));
      SB_CUDA(cudaMemcpyAsync(g->pt_bits.p, bp.data(), (size_t)n1 * 8, cudaMemcpyHostToDevice, s));
      if (!units.empty()) {
        SB_CUDA(cudaMemcpyAsync(g->a3_units.p, units.data(), units.size() * sizeof(AUnit), cudaMemcpyHostToDevice, s));
        A3Params A;
        memset(&A, 0, sizeof(A));
        seg_view(g, A.S); A.a128 = g->a_post.p; A.t_aoff = g->t_aoff.p;
        A.q_terms = g->q_terms.p; A.q_nterms = g->q_nterms.p; A.q_weights = g->q_weights.p; A.n_terms_max = 1;
        A.units = (const AUnit*)g->a3_units.p; A.n_units = (uint32_t)units.size(); A.counters = g->counters.p;
        SB_TRY(timed([&]() -> int { SB_LAUNCH(k_docset_postings, div_up(A.n_units, A3_WARPS), A3_WARPS * 32, 0, s, A, (uint32_t* const*)g->pt_bits.p); SB_CHECK_LAUNCH(); return SB200_OK; }));
      }
      SB_CUDA(cudaStreamSynchronize(s));   // the host tables above are reused by the positional patterns
    }
    // positional patterns
    std::vector<uint32_t> nq_p;
    for (uint32_t p = 0; p < np_; p++) if (kind[p] == NORMAL) nq_p.push_back(p);
    const uint32_t nq = (uint32_t)nq_p.size(), nt = std::max<uint32_t>(NT, 1), npw = std::max<uint32_t>(NP, 1);
    if (nq) {
      std::vector<uint32_t> terms((size_t)nq * nt, 0), col((size_t)nq * nt, 0), nt_q(nq, 0), np_q(nq, 0);
      std::vector<uint8_t> parts((size_t)nq * npw, 0);
      for (uint32_t i = 0; i < nq; i++) {
        const uint32_t p = nq_p[i], c = nterms[p];
        uint32_t idx[MAXT];
        for (uint32_t j = 0; j < c; j++) idx[j] = j;
        const uint32_t* ords = b->term_ords + (size_t)p * NT;
        std::stable_sort(idx, idx + c, [&](uint32_t x, uint32_t y) { return g->h_df[ords[x]] < g->h_df[ords[y]]; });
        for (uint32_t r = 0; r < c; r++) { terms[(size_t)i * nt + r] = ords[idx[r]]; col[(size_t)i * nt + idx[r]] = r; }
        for (uint32_t j = 0; j < nparts[p]; j++) parts[(size_t)i * npw + j] = b->parts[(size_t)p * NP + j];
        nt_q[i] = c; np_q[i] = nparts[p];
        bp[i] = (uint64_t)(uintptr_t)out[p]->bits.p;
      }
      SB_TRY(ensure(g->q_terms, terms.size())); SB_TRY(ensure(g->pt_col, col.size())); SB_TRY(ensure(g->q_nterms, nq));
      SB_TRY(ensure(g->pt_nparts, nq)); SB_TRY(ensure(g->pt_parts, parts.size()));
      SB_TRY(ensure(g->a3_off, nq)); SB_TRY(ensure(g->a3_cnt, nq)); SB_TRY(ensure(g->ph_ovc, 4)); SB_TRY(ensure(g->ph_pre, (size_t)nq + 1));
      SB_CUDA(cudaMemcpyAsync(g->q_terms.p, terms.data(), terms.size() * 4, cudaMemcpyHostToDevice, s));
      SB_CUDA(cudaMemcpyAsync(g->pt_col.p, col.data(), col.size() * 4, cudaMemcpyHostToDevice, s));
      SB_CUDA(cudaMemcpyAsync(g->q_nterms.p, nt_q.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, s));
      SB_CUDA(cudaMemcpyAsync(g->pt_nparts.p, np_q.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, s));
      SB_CUDA(cudaMemcpyAsync(g->pt_parts.p, parts.data(), parts.size(), cudaMemcpyHostToDevice, s));
      SB_CUDA(cudaMemcpyAsync(g->pt_bits.p, bp.data(), (size_t)nq * 8, cudaMemcpyHostToDevice, s));
      SB_CUDA(cudaMemsetAsync(g->a3_cnt.p, 0, (size_t)nq * 4, s));
      const size_t cand_smem = (size_t)A3_WARPS * nt * 128 * 12;
      static size_t cand_conf = 0;
      if (cand_conf < cand_smem) { SB_CUDA(cudaFuncSetAttribute(k_phrase_cand<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cand_smem)); cand_conf = cand_smem; }
      int n_sm = 132;
      { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev); if (n_sm <= 0) n_sm = 132; }
      uint64_t budget = (uint64_t)2 << 30;   // candidate records: doc + nt x (u64 offset, u32 tf)
      const uint64_t max_entries = std::max<uint64_t>(budget / (4 + 12 * (uint64_t)nt), 1);
      std::vector<uint64_t> off(nq, 0), pre(nq + 1, 0);
      std::vector<uint32_t> cnt(nq, 0);
      std::vector<AUnit> units;
      uint32_t g0 = 0;
      while (g0 < nq) {
        uint64_t entries = 0; uint32_t g1 = g0;
        units.clear();
        while (g1 < nq) {
          const uint32_t dfA = g->h_df[terms[(size_t)g1 * nt]];
          if (g1 > g0 && entries + dfA > max_entries) break;
          off[g1] = entries; entries += dfA;
          const uint32_t nblk = (dfA >> 7) + ((dfA & 127u) ? 1u : 0u);
          for (uint32_t b0 = 0; b0 < nblk; b0 += A3_UNIT_BLOCKS) { AUnit u; u.q = g1; u.blk_lo = b0; u.blk_hi = std::min(nblk, b0 + A3_UNIT_BLOCKS); u._pad = 0; units.push_back(u); }
          g1++;
        }
        const uint32_t n_units = (uint32_t)units.size();
        const size_t ne = (size_t)std::max<uint64_t>(entries, 1);
        SB_TRY(ensure(g->ph_cdoc, ne)); SB_TRY(ensure(g->ph_coff, ne * nt)); SB_TRY(ensure(g->ph_ctf, ne * nt));
        SB_TRY(ensure(g->a3_units, std::max<size_t>(n_units, 1)));
        SB_CUDA(cudaMemcpyAsync(g->a3_off.p + g0, off.data() + g0, (size_t)(g1 - g0) * 8, cudaMemcpyHostToDevice, s));
        if (n_units) {
          SB_CUDA(cudaMemcpyAsync(g->a3_units.p, units.data(), (size_t)n_units * sizeof(AUnit), cudaMemcpyHostToDevice, s));
          PhCandParams C;
          memset(&C, 0, sizeof(C));
          seg_view(g, C.A.S); C.A.a128 = g->a_post.p; C.A.t_aoff = g->t_aoff.p;
          C.A.q_terms = g->q_terms.p; C.A.q_nterms = g->q_nterms.p; C.A.q_weights = g->q_weights.p; C.A.n_terms_max = nt;
          C.A.units = (const AUnit*)g->a3_units.p; C.A.n_units = n_units;
          C.A.cand_off = g->a3_off.p; C.A.cand_cnt = g->a3_cnt.p; C.A.counters = g->counters.p;
          C.pos_base = g->pos_base.p; C.nt = nt; C.c_doc = g->ph_cdoc.p; C.c_off = g->ph_coff.p; C.c_tf = g->ph_ctf.p;
          SB_TRY(timed([&]() -> int { SB_LAUNCH(k_phrase_cand<1>, div_up(n_units, A3_WARPS), A3_WARPS * 32, cand_smem, s, C); SB_CHECK_LAUNCH(); return SB200_OK; }));
        }
        SB_CUDA(cudaMemcpyAsync(cnt.data() + g0, g->a3_cnt.p + g0, (size_t)(g1 - g0) * 4, cudaMemcpyDeviceToHost, s));
        SB_CUDA(cudaStreamSynchronize(s));
        const uint32_t ns = g1 - g0;
        pre[0] = 0;
        for (uint32_t i = 0; i < ns; i++) pre[i + 1] = pre[i] + cnt[g0 + i];
        const uint64_t total = pre[ns];
        if (total) {
          SB_CUDA(cudaMemcpyAsync(g->ph_pre.p, pre.data(), (size_t)(ns + 1) * 8, cudaMemcpyHostToDevice, s));
          SB_TRY(ensure(g->ph_ov, (size_t)total));
          PtParams V;
          memset(&V, 0, sizeof(V));
          pos_view(g, V.V);
          V.q_terms = g->q_terms.p; V.q_col = g->pt_col.p; V.q_parts = g->pt_parts.p; V.q_nparts = g->pt_nparts.p; V.q_nterms = g->q_nterms.p;
          V.nt = nt; V.np = npw; V.token_counts = g->has_tok ? g->tok_count.p : nullptr;
          V.cand_off = g->a3_off.p; V.cand_pre = g->ph_pre.p; V.slot0 = g0; V.n_slots = ns;
          V.c_doc = g->ph_cdoc.p; V.c_off = g->ph_coff.p; V.c_tf = g->ph_ctf.p;
          V.q_bits = (uint32_t* const*)g->pt_bits.p; V.counters = g->counters.p;
          V.list = nullptr; V.n = total; V.ov_list = (unsigned long long*)g->ph_ov.p; V.ov = g->ph_ovc.p; V.scratch_cursor = g->ph_ovc.p + 2;
          SB_CUDA(cudaMemsetAsync(g->ph_ovc.p, 0, 4 * sizeof(unsigned long long), s));
          const unsigned grid = (unsigned)std::min<uint64_t>(div_up(total, PT_WARPS), (uint64_t)n_sm * 16);
          SB_TRY(timed([&]() -> int { SB_LAUNCH(k_pattern_verify, grid, PT_WARPS * 32, 0, s, V); SB_CHECK_LAUNCH(); return SB200_OK; }));
          // candidates whose lists do not fit shared memory: one pass over global scratch (chains only shrink)
          unsigned long long ov[4] = {0, 0, 0, 0};
          SB_CUDA(cudaMemcpyAsync(ov, g->ph_ovc.p, sizeof(ov), cudaMemcpyDeviceToHost, s));
          SB_CUDA(cudaStreamSynchronize(s));
          if (ov[0]) {
            SB_TRY(ensure(g->ph_scratch, (size_t)(ov[1] + 64)));
            V.list = (const unsigned long long*)g->ph_ov.p; V.n = ov[0]; V.ov_list = nullptr; V.scratch = g->ph_scratch.p;
            SB_CUDA(cudaMemsetAsync(g->ph_ovc.p, 0, 4 * sizeof(unsigned long long), s));
            const unsigned grid2 = (unsigned)std::min<uint64_t>(div_up(ov[0], PT_WARPS), (uint64_t)n_sm * 16);
            SB_TRY(timed([&]() -> int { SB_LAUNCH(k_pattern_verify, grid2, PT_WARPS * 32, 0, s, V); SB_CHECK_LAUNCH(); return SB200_OK; }));
          }
        }
        g0 = g1;
      }
    }
    unsigned long long h[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    SB_CUDA(cudaMemcpyAsync(h, g->counters.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaEventRecord(g->ev1, s));
    SB_CUDA(cudaStreamSynchronize(s));
    if (h[2]) SB_FAIL(SB200_EFORMAT, "%llu pattern work items met inconsistent posting / position data", h[2]);
    if (stats) {
      stats->candidates = h[0]; stats->matches = h[1]; stats->positions_decoded = h[3]; stats->position_bytes = h[4];
      cudaEventElapsedTime(&stats->ms, g->ev0, g->ev1); stats->kernel_ms = kms;
    }
    return SB200_OK;
  }();
  if (rc != SB200_OK) return fail_cleanup(rc);
  return SB200_OK;
}

}  // namespace sb200
using namespace sb200;

namespace sb200 {
// TermInfoStore::get for every term ordinal (tantivy/src/termdict/fst_termdict/term_info_store.rs:55-99,134-153): the
// block's first TermInfo comes verbatim from its 47-byte TermInfoBlockMeta, the other 255 are bit-packed offsets
// relative to it, read with the reference's unaligned little-endian 8-byte window (:102-122).
__device__ __forceinline__ uint64_t tis_u64(const uint8_t* p, uint64_t avail) {
  uint64_t v = 0;
  for (uint32_t i = 0; i < 8u && i < avail; i++) v |= (uint64_t)p[i] << (8u * i);
  return v;
}
__device__ __forceinline__ uint64_t tis_bits(const uint8_t* data, uint64_t len, uint64_t addr_bits, uint32_t nb) {
  const uint64_t ab = addr_bits >> 3;
  if (ab >= len) return 0;
  const uint64_t v = tis_u64(data + ab, len - ab) >> (addr_bits & 7u);
  return v & ((1ull << nb) - 1ull);
}
__global__ void k_term_info_store(const uint8_t* __restrict__ file, uint64_t len, uint64_t meta_len, uint64_t n_terms,
                                  sb200_term_info* out, int* err) {
  const uint64_t ord = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (ord >= n_terms) return;
  const uint8_t* m = file + 16 + (ord >> 8) * 47;
  const uint8_t* infos = file + 16 + meta_len;
  const uint64_t infos_len = len - 16 - meta_len;
  const uint64_t off = tis_u64(m, 8);
  const uint32_t rdf = (uint32_t)tis_u64(m + 8, 4);
  const uint64_t rps = tis_u64(m + 12, 8), rpl = tis_u64(m + 20, 8);
  const uint32_t dfb = m[44], pb = m[45], qb = m[46];
  const uint32_t inner = (uint32_t)(ord & 255u);
  sb200_term_info ti; ti._pad = 0;
  if (inner == 0) { ti.postings_off = rps; ti.postings_len = rpl; ti.doc_freq = rdf; }
  else {
    if (off > infos_len || dfb > 56 || pb > 56 || qb > 56) { *err = 1; return; }
    const uint64_t nb = (uint64_t)dfb + pb + qb, a0 = nb * (inner - 1);
    const uint8_t* d = infos + off; const uint64_t dl = infos_len - off;
    const uint64_t ps = rps + tis_bits(d, dl, a0, pb), pe = rps + tis_bits(d, dl, a0 + nb, pb);
    if (pe < ps) { *err = 2; return; }
    ti.postings_off = ps; ti.postings_len = pe - ps;
    ti.doc_freq = (uint32_t)tis_bits(d, dl, a0 + pb + qb, dfb);
  }
  out[ord] = ti;
}
// TermInfo.positions_range of every ordinal (term_info_store.rs:63-91): the block's reference range sits after its postings
// range in the TermInfoBlockMeta (TermInfo::serialize, term_info.rs:41-47), the bit-packed start follows the postings start
__global__ void k_term_info_store_positions(const uint8_t* __restrict__ file, uint64_t len, uint64_t meta_len, uint64_t n_terms,
                                            uint64_t* pos_off, uint64_t* pos_len, int* err) {
  const uint64_t ord = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (ord >= n_terms) return;
  const uint8_t* m = file + 16 + (ord >> 8) * 47;
  const uint8_t* infos = file + 16 + meta_len;
  const uint64_t infos_len = len - 16 - meta_len;
  const uint64_t off = tis_u64(m, 8);
  const uint64_t rqs = tis_u64(m + 28, 8), rql = tis_u64(m + 36, 8);
  const uint32_t dfb = m[44], pb = m[45], qb = m[46];
  const uint32_t inner = (uint32_t)(ord & 255u);
  uint64_t s = rqs, l = rql;
  if (inner != 0) {
    if (off > infos_len || dfb > 56 || pb > 56 || qb > 56) { *err = 1; return; }
    const uint64_t nb = (uint64_t)dfb + pb + qb, a0 = nb * (inner - 1) + pb;
    const uint8_t* d = infos + off; const uint64_t dl = infos_len - off;
    const uint64_t qs = rqs + tis_bits(d, dl, a0, qb), qe = rqs + tis_bits(d, dl, a0 + nb, qb);
    if (qe < qs) { *err = 2; return; }
    s = qs; l = qe - qs;
  }
  pos_off[ord] = s; pos_len[ord] = l;
}
}  // namespace sb200

extern "C" {

int sb200_term_info_store_decode(const uint8_t* store, uint64_t len, int device, sb200_term_info* infos, uint64_t cap,
                                 uint64_t* n_terms) {
  using namespace sb200;
  if (!store || !n_terms) SB_FAIL(SB200_EINVAL, "NULL argument");
  if (len < 16) SB_FAIL(SB200_EFORMAT, "term info store shorter than its 16-byte header");
  SB_CUDA(cudaSetDevice(device));
  uint8_t head[16];
  SB_CUDA(cudaMemcpy(head, store, 16, cudaMemcpyDefault));
  uint64_t meta_len = 0, n = 0;
  memcpy(&meta_len, head, 8); memcpy(&n, head + 8, 8);
  if (meta_len > len - 16 || meta_len != 47ull * ((n + 255) / 256)) SB_FAIL(SB200_EFORMAT, "term info store: %llu terms need %llu bytes of block metadata, header says %llu", (unsigned long long)n, (unsigned long long)(47ull * ((n + 255) / 256)), (unsigned long long)meta_len);
  *n_terms = n;
  const uint64_t k = std::min<uint64_t>(n, cap);
  if (!infos || k == 0) return SB200_OK;
  DevBuf<uint8_t> d_store; DevBuf<sb200_term_info> d_out; DevBuf<int> d_err;
  SB_TRY(d_store.alloc(len)); SB_TRY(d_out.alloc(n)); SB_TRY(d_err.alloc(1));
  SB_CUDA(cudaMemcpy(d_store.p, store, len, cudaMemcpyDefault));
  SB_CUDA(cudaMemset(d_err.p, 0, sizeof(int)));
  SB_LAUNCH(k_term_info_store, div_up(n, 256), 256, 0, (cudaStream_t)0, d_store.p, len, meta_len, n, d_out.p, d_err.p);
  SB_CHECK_LAUNCH();
  int h_err = 0;
  SB_CUDA(cudaMemcpy(&h_err, d_err.p, sizeof(int), cudaMemcpyDeviceToHost));
  if (h_err) SB_FAIL(SB200_EFORMAT, "term info store is inconsistent (code %d)", h_err);
  SB_CUDA(cudaMemcpy(infos, d_out.p, k * sizeof(sb200_term_info), cudaMemcpyDefault));
  return SB200_OK;
}

int sb200_term_info_store_decode_positions(const uint8_t* store, uint64_t len, int device, uint64_t* positions_off, uint64_t* positions_len,
                                           uint64_t cap, uint64_t* n_terms) {
  using namespace sb200;
  if (!store || !n_terms) SB_FAIL(SB200_EINVAL, "NULL argument");
  if (len < 16) SB_FAIL(SB200_EFORMAT, "term info store shorter than its 16-byte header");
  SB_CUDA(cudaSetDevice(device));
  uint8_t head[16];
  SB_CUDA(cudaMemcpy(head, store, 16, cudaMemcpyDefault));
  uint64_t meta_len = 0, n = 0;
  memcpy(&meta_len, head, 8); memcpy(&n, head + 8, 8);
  if (meta_len > len - 16 || meta_len != 47ull * ((n + 255) / 256)) SB_FAIL(SB200_EFORMAT, "term info store: %llu terms need %llu bytes of block metadata, header says %llu", (unsigned long long)n, (unsigned long long)(47ull * ((n + 255) / 256)), (unsigned long long)meta_len);
  *n_terms = n;
  const uint64_t k = std::min<uint64_t>(n, cap);
  if (!positions_off || !positions_len || k == 0) return SB200_OK;
  DevBuf<uint8_t> d_store; DevBuf<uint64_t> d_off, d_len; DevBuf<int> d_err;
  SB_TRY(d_store.alloc(len)); SB_TRY(d_off.alloc(n)); SB_TRY(d_len.alloc(n)); SB_TRY(d_err.alloc(1));
  SB_CUDA(cudaMemcpy(d_store.p, store, len, cudaMemcpyDefault));
  SB_CUDA(cudaMemset(d_err.p, 0, sizeof(int)));
  SB_LAUNCH(k_term_info_store_positions, div_up(n, 256), 256, 0, (cudaStream_t)0, d_store.p, len, meta_len, n, d_off.p, d_len.p, d_err.p);
  SB_CHECK_LAUNCH();
  int h_err = 0;
  SB_CUDA(cudaMemcpy(&h_err, d_err.p, sizeof(int), cudaMemcpyDeviceToHost));
  if (h_err) SB_FAIL(SB200_EFORMAT, "term info store is inconsistent (code %d)", h_err);
  SB_CUDA(cudaMemcpy(positions_off, d_off.p, k * 8, cudaMemcpyDefault));
  SB_CUDA(cudaMemcpy(positions_len, d_len.p, k * 8, cudaMemcpyDefault));
  return SB200_OK;
}

int sb200_segment_create(const uint8_t* postings_file, uint64_t postings_len, const sb200_term_info* terms, uint32_t n_terms,
                         const uint8_t* fieldnorm_ids, uint32_t max_doc, int record_option, int device, sb200_segment** out) {
  if (!out) SB_FAIL(SB200_EINVAL, "out is NULL");
  *out = nullptr;
  if ((postings_len && !postings_file) || (n_terms && !terms) || (max_doc && !fieldnorm_ids)) SB_FAIL(SB200_EINVAL, "NULL argument");
  if (record_option < 0 || record_option > 2) SB_FAIL(SB200_EINVAL, "record_option %d", record_option);
  if (max_doc >= TERMINATED) SB_FAIL(SB200_ERANGE, "max_doc must be < 2^31-1 (TERMINATED, tantivy/src/docset.rs:9)");
  int ndev = 0;
  SB_CUDA(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) SB_FAIL(SB200_EINVAL, "device %d not in [0,%d)", device, ndev);
  SB_CUDA(cudaSetDevice(device));
  sb200_segment* g = new (std::nothrow) sb200_segment();
  if (!g) SB_FAIL(SB200_ENOMEM, "host allocation failed");
  g->device = device; g->record = record_option; g->stride = record_option == 0 ? 5 : (record_option == 1 ? 8 : 12);
  g->max_doc = max_doc; g->n_terms = n_terms; g->postings_len = postings_len;
  auto body = [&]() -> int {
    SB_CUDA(cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking));
    SB_CUDA(cudaEventCreate(&g->ev0)); SB_CUDA(cudaEventCreate(&g->ev1));
    SB_CUDA(cudaEventCreate(&g->evk0)); SB_CUDA(cudaEventCreate(&g->evk1));
    cudaStream_t s = g->stream;
    SB_CUDA(cudaEventRecord(g->ev0, s));
    SB_TRY(g->postings.alloc(postings_len + 64));
    SB_CUDA(cudaMemsetAsync(g->postings.p + postings_len, 0, 64, s));
    SB_TRY(copy_in(g->postings.p, postings_file, postings_len, s));
    SB_TRY(g->fieldnorm.alloc((size_t)max_doc + 16));
    SB_TRY(copy_in(g->fieldnorm.p, fieldnorm_ids, max_doc, s));
    // block slots: n_full + 1 per term (the extra one records where the vint tail starts)
    std::vector<sb200_term_info> h_terms;
    const sb200_term_info* ht = terms;
    if (n_terms && is_device_ptr(terms)) { h_terms.resize(n_terms); SB_CUDA(cudaMemcpy(h_terms.data(), terms, (size_t)n_terms * sizeof(sb200_term_info), cudaMemcpyDeviceToHost)); ht = h_terms.data(); }
    std::vector<uint32_t> first(n_terms + 1);
    g->h_df.resize(n_terms);
    uint64_t slots = 0, postings = 0;
    for (uint32_t t = 0; t < n_terms; t++) {
      first[t] = (uint32_t)slots; slots += (ht[t].doc_freq >> 7) + 1; g->h_df[t] = ht[t].doc_freq; postings += ht[t].doc_freq;
      if (slots >= 0xFFFFFFF0ull) SB_FAIL(SB200_ERANGE, "more than 2^32 posting blocks");
      if (ht[t].postings_len >= 0xFFFFFFFFull) SB_FAIL(SB200_ERANGE, "term %u: posting list larger than 4 GiB", t);
    }
    first[n_terms] = (uint32_t)slots;
    g->n_blocks = slots - n_terms; g->n_postings = postings;
    SB_TRY(g->t_first.alloc(n_terms + 1)); SB_TRY(g->t_data_off.alloc(n_terms + 1)); SB_TRY(g->t_end_off.alloc(n_terms + 1)); SB_TRY(g->t_df.alloc(n_terms + 1));
    SB_TRY(g->b_last.alloc(slots + 1)); SB_TRY(g->b_off.alloc(slots + 1)); SB_TRY(g->b_bits.alloc(slots + 1)); SB_TRY(g->b_bw.alloc(slots + 1));
    SB_CUDA(cudaMemcpyAsync(g->t_first.p, first.data(), (size_t)(n_terms + 1) * 4, cudaMemcpyHostToDevice, s));
    DevBuf<sb200_term_info> d_terms; DevBuf<int> d_err;
    SB_TRY(d_terms.alloc(n_terms + 1)); SB_TRY(d_err.alloc(1));
    SB_CUDA(cudaMemcpyAsync(d_terms.p, ht, (size_t)n_terms * sizeof(sb200_term_info), cudaMemcpyHostToDevice, s));
    SB_CUDA(cudaMemsetAsync(d_err.p, 0, sizeof(int), s));
    if (n_terms) {
      SB_LAUNCH(k_build_directory, div_up((uint64_t)n_terms * 32, 256), 256, 0, s, g->postings.p, d_terms.p, n_terms, g->stride,
                g->t_first.p, g->t_data_off.p, g->t_end_off.p, g->t_df.p, g->b_last.p, g->b_off.p, g->b_bits.p, g->b_bw.p, postings_len, d_err.p);
      SB_CHECK_LAUNCH();
    }
    int h_err = 0;
    SB_CUDA(cudaMemcpyAsync(&h_err, d_err.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    SB_CUDA(cudaStreamSynchronize(s));
    if (h_err) SB_FAIL(SB200_EFORMAT, "malformed postings (code %d): term range outside the file, skip length != blocks x %d, or bit width > 32", h_err, g->stride);
    // aligned copy of the block regions: per-term size (uint4 units) -> exclusive scan -> realigning copy
    SB_TRY(g->t_aoff.alloc(n_terms + 1));
    uint64_t total_units = 0;
    if (n_terms) {
      DevBuf<uint64_t> units; SB_TRY(units.alloc(n_terms + 1));
      SB_CUDA(cudaMemsetAsync(units.p + n_terms, 0, 8, s));
      SB_LAUNCH(k_block_units, div_up(n_terms, 256), 256, 0, s, g->t_first.p, g->t_df.p, g->b_off.p, n_terms, units.p);
      SB_CHECK_LAUNCH();
      size_t need = 0;
      SB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, need, units.p, g->t_aoff.p, (int64_t)(n_terms + 1), s));
      DevBuf<uint8_t> tmp; SB_TRY(tmp.alloc(need + 256));
      SB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, need, units.p, g->t_aoff.p, (int64_t)(n_terms + 1), s));
      g_launches.fetch_add(2, std::memory_order_relaxed);
      SB_CUDA(cudaMemcpyAsync(&total_units, g->t_aoff.p + n_terms, 8, cudaMemcpyDeviceToHost, s));
      SB_CUDA(cudaStreamSynchronize(s));
    }
    SB_TRY(g->a_post.alloc(total_units + 4));
    if (n_terms && total_units) {
      SB_LAUNCH(k_align_blocks, div_up((uint64_t)n_terms * 32, 256), 256, 0, s, (const uint32_t*)g->postings.p, g->t_data_off.p,
                g->t_first.p, g->t_df.p, g->b_off.p, g->t_aoff.p, n_terms, (uint32_t*)g->a_post.p);
      SB_CHECK_LAUNCH();
    }
    SB_CUDA(cudaEventRecord(g->ev1, s));
    SB_CUDA(cudaStreamSynchronize(s));
    float ms = 0; cudaEventElapsedTime(&ms, g->ev0, g->ev1); g->stage_ms = ms;
    return SB200_OK;
  };
  const int rc = body();
  if (rc != SB200_OK) { sb200_segment_destroy(g); return rc; }
  *out = g;
  return SB200_OK;
}

void sb200_segment_destroy(sb200_segment* g) {
  if (!g) return;
  cudaSetDevice(g->device);
  if (g->stream) cudaStreamSynchronize(g->stream);
  if (g->ev0) cudaEventDestroy(g->ev0);
  if (g->ev1) cudaEventDestroy(g->ev1);
  if (g->evk0) cudaEventDestroy(g->evk0);
  if (g->evk1) cudaEventDestroy(g->evk1);
  if (g->h_pack) cudaFreeHost(g->h_pack);
  cudaStream_t s = g->stream;
  delete g;
  if (s) cudaStreamDestroy(s);
}

int sb200_segment_get_info(const sb200_segment* g, sb200_segment_info* info) {
  if (!g || !info) SB_FAIL(SB200_EINVAL, "NULL argument");
  info->n_terms = g->n_terms; info->n_blocks = g->n_blocks; info->n_postings = g->n_postings; info->max_doc = g->max_doc; info->_pad = 0;
  info->hbm_bytes = g->postings.bytes() + g->fieldnorm.bytes() + g->t_first.bytes() + g->t_data_off.bytes() + g->t_end_off.bytes() +
                    g->t_df.bytes() + g->b_last.bytes() + g->b_off.bytes() + g->b_bits.bytes() + g->b_bw.bytes();
  if (g->has_pos)
    info->hbm_bytes += g->pos_file.bytes() + g->pos_data_off.bytes() + g->pos_tail_off.bytes() + g->pos_end_off.bytes() + g->pos_count.bytes() +
                       g->pos_first.bytes() + g->pos_nblk.bytes() + g->pos_b_off.bytes() + g->pos_b_w.bytes() + g->pos_base.bytes();
  info->stage_ms = g->stage_ms;
  return SB200_OK;
}

int sb200_signals_create(const double* const* columns, uint32_t n_cols, uint32_t max_doc, int device, sb200_signals** out) {
  if (!out) SB_FAIL(SB200_EINVAL, "out is NULL");
  *out = nullptr;
  if (n_cols && !columns) SB_FAIL(SB200_EINVAL, "columns is NULL");
  if (n_cols > 64) SB_FAIL(SB200_ERANGE, "at most 64 signal columns");
  SB_CUDA(cudaSetDevice(device));
  sb200_signals* sg = new (std::nothrow) sb200_signals();
  if (!sg) SB_FAIL(SB200_ENOMEM, "host allocation failed");
  sg->device = device; sg->n_cols = n_cols; sg->max_doc = max_doc;
  auto body = [&]() -> int {
    if (!n_cols || !max_doc) return SB200_OK;
    SB_TRY(sg->rows.alloc((size_t)max_doc * n_cols));
    std::vector<DevBuf<double>> tmp(n_cols);
    std::vector<const double*> ptrs(n_cols);
    for (uint32_t c = 0; c < n_cols; c++) {
      if (!columns[c]) SB_FAIL(SB200_EINVAL, "column %u is NULL", c);
      if (is_device_ptr(columns[c])) ptrs[c] = columns[c];
      else { SB_TRY(tmp[c].alloc(max_doc)); SB_CUDA(cudaMemcpy(tmp[c].p, columns[c], (size_t)max_doc * 8, cudaMemcpyHostToDevice)); ptrs[c] = tmp[c].p; }
    }
    DevBuf<const double*> d_ptrs; SB_TRY(d_ptrs.alloc(n_cols));
    SB_CUDA(cudaMemcpy(d_ptrs.p, ptrs.data(), n_cols * sizeof(double*), cudaMemcpyHostToDevice));
    SB_LAUNCH(k_interleave_signals, div_up((uint64_t)max_doc * n_cols, 256), 256, 0, 0, d_ptrs.p, n_cols, max_doc, sg->rows.p);
    SB_CHECK_LAUNCH();
    SB_CUDA(cudaDeviceSynchronize());
    return SB200_OK;
  };
  const int rc = body();
  if (rc != SB200_OK) { delete sg; return rc; }
  *out = sg;
  return SB200_OK;
}
int sb200_signals_create_raw(const sb200_numeric_column* cols, uint32_t n_cols, uint32_t max_doc, int device, sb200_signals** out) {
  if (!out) SB_FAIL(SB200_EINVAL, "out is NULL");
  *out = nullptr;
  if (n_cols && !cols) SB_FAIL(SB200_EINVAL, "cols is NULL");
  if (n_cols > 64) SB_FAIL(SB200_ERANGE, "at most 64 signal columns");
  SB_CUDA(cudaSetDevice(device));
  sb200_signals* sg = new (std::nothrow) sb200_signals();
  if (!sg) SB_FAIL(SB200_ENOMEM, "host allocation failed");
  sg->device = device; sg->n_cols = n_cols; sg->max_doc = max_doc;
  auto body = [&]() -> int {
    if (!n_cols || !max_doc) return SB200_OK;
    SB_TRY(sg->rows.alloc((size_t)max_doc * n_cols));
    for (uint32_t c = 0; c < n_cols; c++) {
      const sb200_numeric_column& col = cols[c];
      if (!col.raw) SB_FAIL(SB200_EINVAL, "column %u: raw is NULL", c);
      if (col.dtype > SB200_NUM_BOOL8) SB_FAIL(SB200_EINVAL, "column %u: unknown dtype %u", c, col.dtype);
      if (col.kind > SB200_NUM_REGION) SB_FAIL(SB200_EINVAL, "column %u: unknown transform %u", c, col.kind);
      const size_t esz = col.dtype == SB200_NUM_BOOL8 ? 1 : 8;
      DevBuf<uint8_t> d_raw; DevBuf<double> d_lut;
      if (col.kind == SB200_NUM_RANK) {
        // score_rank = (10 - (1 + rank).log(8)).max(0) (non_text.rs:50-59), f64::log(base) = ln(x) / ln(base).  `ln` is the host
        // C library's (as for a Rust binary on the same machine); no device `log` is bit-identical to it, so this one transform
        // is evaluated on the host at open time and only the finished column crosses PCIe.
        if (col.dtype != SB200_NUM_U64) SB_FAIL(SB200_EINVAL, "column %u: score_rank reads a u64 column", c);
        std::vector<uint64_t> h_raw;
        const uint64_t* r = (const uint64_t*)col.raw;
        if (is_device_ptr(col.raw)) { h_raw.resize(max_doc); SB_CUDA(cudaMemcpy(h_raw.data(), col.raw, (size_t)max_doc * 8, cudaMemcpyDeviceToHost)); r = h_raw.data(); }
        std::vector<double> sc(max_doc);
        const double ln8 = log(8.0);
        for (uint32_t d = 0; d < max_doc; d++) { const double v = 10.0 - log(1.0 + (double)r[d]) / ln8; sc[d] = v > 0.0 ? v : 0.0; }
        SB_TRY(d_raw.alloc((size_t)max_doc * 8));
        SB_CUDA(cudaMemcpy(d_raw.p, sc.data(), (size_t)max_doc * 8, cudaMemcpyHostToDevice));
        SB_LAUNCH(k_numeric_score, div_up(max_doc, 256), 256, 0, 0, (uint32_t)SB200_NUM_IDENTITY, (uint32_t)SB200_NUM_F64, (const void*)d_raw.p, max_doc, 0.0, 0.0,
                  (const double*)nullptr, 0u, sg->rows.p, n_cols, c);
        SB_CHECK_LAUNCH();
        SB_CUDA(cudaDeviceSynchronize());
        continue;
      }
      const void* raw = col.raw;
      if (!is_device_ptr(col.raw)) {
        SB_TRY(d_raw.alloc((size_t)max_doc * esz));
        SB_CUDA(cudaMemcpy(d_raw.p, col.raw, (size_t)max_doc * esz, cudaMemcpyHostToDevice));
        raw = d_raw.p;
      }
      const double* lut = nullptr;
      if (col.kind == SB200_NUM_REGION && col.lut && col.lut_len) {
        SB_TRY(d_lut.alloc(col.lut_len));
        SB_CUDA(cudaMemcpy(d_lut.p, col.lut, (size_t)col.lut_len * 8, cudaMemcpyDefault));
        lut = d_lut.p;
      }
      SB_LAUNCH(k_numeric_score, div_up(max_doc, 256), 256, 0, 0, col.kind, col.dtype, raw, max_doc, col.p0, col.p1, lut, lut ? col.lut_len : 0u,
                sg->rows.p, n_cols, c);
      SB_CHECK_LAUNCH();
      SB_CUDA(cudaDeviceSynchronize());   // the staging copies of this column are released at the end of the iteration
    }
    return SB200_OK;
  };
  const int rc = body();
  if (rc != SB200_OK) { delete sg; return rc; }
  *out = sg;
  return SB200_OK;
}
int sb200_signals_read(const sb200_signals* s, uint32_t first_doc, uint32_t n_docs, double* rows_out) {
  if (!s || (!rows_out && n_docs)) SB_FAIL(SB200_EINVAL, "NULL argument");
  if ((uint64_t)first_doc + n_docs > s->max_doc) SB_FAIL(SB200_ERANGE, "docs [%u, +%u) outside the table of %u", first_doc, n_docs, s->max_doc);
  SB_CUDA(cudaSetDevice(s->device));
  if (n_docs && s->n_cols)
    SB_CUDA(cudaMemcpy(rows_out, s->rows.p + (size_t)first_doc * s->n_cols, (size_t)n_docs * s->n_cols * 8, cudaMemcpyDeviceToHost));
  return SB200_OK;
}
void sb200_signals_destroy(sb200_signals* s) {
  if (!s) return;
  cudaSetDevice(s->device);
  delete s;
}

int sb200_bm25_topk_batch(sb200_segment* seg, const sb200_bm25_batch* batch, uint32_t* docs, float* scores, uint32_t* n_out,
                          sb200_bm25_stats* stats) {
  if (!seg) SB_FAIL(SB200_EINVAL, "NULL segment handle");
  SB_CUDA(cudaSetDevice(seg->device));
  if (!scores) SB_FAIL(SB200_EINVAL, "scores is NULL");
  if (!batch) SB_FAIL(SB200_EINVAL, "batch is NULL");
  return run_batch(seg, batch, batch->mode, nullptr, docs, scores, nullptr, n_out, stats);
}

int sb200_bm25_topk(sb200_segment* seg, const uint32_t* term_ords, const float* weights, uint32_t n_terms, const float* tf_cache256,
                    int mode, uint32_t k, uint32_t* docs, float* scores, uint32_t* n_out) {
  sb200_bm25_batch b;
  b.n_queries = 1; b.n_terms = n_terms; b.term_ords = term_ords; b.weights = weights; b.tf_cache256 = tf_cache256; b.mode = mode; b.k = k;
  return sb200_bm25_topk_batch(seg, &b, docs, scores, n_out, nullptr);
}

int sb200_segment_attach_positions(sb200_segment* g, const uint8_t* positions_file, uint64_t len, const uint64_t* positions_off,
                                   const uint64_t* positions_len) {
  if (!g) SB_FAIL(SB200_EINVAL, "NULL segment handle");
  if (g->record != SB200_RECORD_FREQS_POSITIONS)
    SB_FAIL(SB200_EINVAL, "the segment was opened with record option %d: positions need WithFreqsAndPositions (2)", g->record);
  const uint32_t n = g->n_terms;
  if ((len && !positions_file) || (n && (!positions_off || !positions_len))) SB_FAIL(SB200_EINVAL, "NULL argument");
  SB_CUDA(cudaSetDevice(g->device));
  g->has_pos = false;
  cudaStream_t s = g->stream;
  std::vector<uint64_t> ho(n), hl(n);
  SB_CUDA(cudaMemcpy(ho.data(), positions_off, (size_t)n * 8, cudaMemcpyDefault));
  SB_CUDA(cudaMemcpy(hl.data(), positions_len, (size_t)n * 8, cudaMemcpyDefault));
  for (uint32_t t = 0; t < n; t++)
    if (ho[t] > len || hl[t] > len - ho[t] || hl[t] == 0) SB_FAIL(SB200_EFORMAT, "term %u: positions range [%llu, +%llu) outside the %llu-byte file or empty", t,
                                                                 (unsigned long long)ho[t], (unsigned long long)hl[t], (unsigned long long)len);
  SB_TRY(g->pos_file.alloc(len + 64));
  SB_CUDA(cudaMemsetAsync(g->pos_file.p + len, 0, 64, s));
  SB_TRY(copy_in(g->pos_file.p, positions_file, len, s));
  DevBuf<uint64_t> d_off, d_len, d_hdr; DevBuf<int> d_err;
  SB_TRY(d_off.alloc(n + 1)); SB_TRY(d_len.alloc(n + 1)); SB_TRY(d_hdr.alloc(n + 1)); SB_TRY(d_err.alloc(1));
  SB_TRY(g->pos_nblk.alloc(n + 1)); SB_TRY(g->pos_first.alloc(n + 1));
  SB_CUDA(cudaMemcpyAsync(d_off.p, ho.data(), (size_t)n * 8, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemcpyAsync(d_len.p, hl.data(), (size_t)n * 8, cudaMemcpyHostToDevice, s));
  SB_CUDA(cudaMemsetAsync(d_err.p, 0, sizeof(int), s));
  std::vector<uint32_t> nblk(n + 1, 0), first(n + 1, 0);
  if (n) {
    SB_LAUNCH(k_pos_header, div_up(n, 256), 256, 0, s, g->pos_file.p, d_off.p, d_len.p, n, g->pos_nblk.p, d_hdr.p, d_err.p);
    SB_CHECK_LAUNCH();
    SB_CUDA(cudaMemcpyAsync(nblk.data(), g->pos_nblk.p, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  }
  int h_err = 0;
  SB_CUDA(cudaMemcpyAsync(&h_err, d_err.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  SB_CUDA(cudaStreamSynchronize(s));
  if (h_err) SB_FAIL(SB200_EFORMAT, "malformed positions: a term's VInt block count is unterminated or exceeds its range");
  uint64_t blocks = 0;
  for (uint32_t t = 0; t < n; t++) {
    first[t] = (uint32_t)blocks; blocks += nblk[t];
    if (blocks >= 0xFFFFFFF0ull) SB_FAIL(SB200_ERANGE, "more than 2^32 positions blocks");
  }
  first[n] = (uint32_t)blocks;
  const uint64_t slots = g->n_blocks + n;   // posting block slots: n_full + 1 per term
  SB_TRY(g->pos_b_off.alloc(blocks + 1)); SB_TRY(g->pos_b_w.alloc(blocks + 1));
  SB_TRY(g->pos_data_off.alloc(n + 1)); SB_TRY(g->pos_tail_off.alloc(n + 1)); SB_TRY(g->pos_end_off.alloc(n + 1)); SB_TRY(g->pos_count.alloc(n + 1));
  SB_TRY(g->pos_base.alloc(slots + 1));
  SB_CUDA(cudaMemcpyAsync(g->pos_first.p, first.data(), (size_t)(n + 1) * 4, cudaMemcpyHostToDevice, s));
  g->h_pos_count.assign(n, 0);
  if (n) {
    SB_LAUNCH(k_pos_dir, div_up((uint64_t)n * 32, 256), 256, 0, s, g->pos_file.p, d_off.p, d_len.p, d_hdr.p, g->pos_nblk.p, g->pos_first.p, n,
              g->postings.p, g->t_data_off.p, g->t_df.p, g->t_first.p, g->pos_data_off.p, g->pos_tail_off.p, g->pos_end_off.p, g->pos_count.p,
              g->pos_b_off.p, g->pos_b_w.p, g->pos_base.p, d_err.p);
    SB_CHECK_LAUNCH();
    SB_CUDA(cudaMemcpyAsync(g->h_pos_count.data(), g->pos_count.p, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
  }
  SB_CUDA(cudaMemcpyAsync(&h_err, d_err.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  SB_CUDA(cudaStreamSynchronize(s));
  if (h_err) SB_FAIL(SB200_EFORMAT, "malformed positions: bit width > 32, blocks beyond the term's range, or a tail that is not a run of < 128 VInts");
  g->has_pos = true;
  return SB200_OK;
}

int sb200_positions_read(sb200_segment* g, uint32_t term, uint64_t offset, uint32_t n, uint32_t* out) {
  if (!g || (n && !out)) SB_FAIL(SB200_EINVAL, "NULL argument");
  if (!g->has_pos) SB_FAIL(SB200_EINVAL, "no positions attached to the segment");
  if (term >= g->n_terms) SB_FAIL(SB200_EINVAL, "term ordinal %u >= %u", term, g->n_terms);
  if (offset > g->h_pos_count[term] || n > g->h_pos_count[term] - offset)
    SB_FAIL(SB200_ERANGE, "positions [%llu, +%u) of term %u: it has %llu", (unsigned long long)offset, n, term, (unsigned long long)g->h_pos_count[term]);
  if (n == 0) return SB200_OK;
  SB_CUDA(cudaSetDevice(g->device));
  DevBuf<uint32_t> tmp;
  uint32_t* dst = out;
  if (!is_device_ptr(out)) { SB_TRY(tmp.alloc(n)); dst = tmp.p; }
  PosView V; pos_view(g, V);
  SB_LAUNCH(k_positions_read, 1, 32, 0, g->stream, V, term, offset, n, dst);
  SB_CHECK_LAUNCH();
  if (dst != out) SB_CUDA(cudaMemcpyAsync(out, dst, (size_t)n * 4, cudaMemcpyDeviceToHost, g->stream));
  SB_CUDA(cudaStreamSynchronize(g->stream));
  return SB200_OK;
}

int sb200_phrase_topk_batch(sb200_segment* seg, const sb200_phrase_batch* batch, uint32_t* docs, float* scores, uint32_t* n_out,
                            sb200_phrase_stats* stats) {
  if (!seg) SB_FAIL(SB200_EINVAL, "NULL segment handle");
  SB_CUDA(cudaSetDevice(seg->device));
  return run_phrase(seg, batch, docs, scores, n_out, stats);
}

int sb200_multi_signal_topk_batch(const sb200_multi_signal_batch* batch, uint32_t* docs, double* totals, uint32_t* n_out,
                                  sb200_bm25_stats* stats) {
  return run_multi(batch, nullptr, docs, totals, n_out, stats);
}
int sb200_signal_topk_batch(sb200_segment* seg, const sb200_signal_batch* batch, uint32_t* docs, double* totals, uint32_t* n_out,
                            sb200_bm25_stats* stats) {
  if (!seg) SB_FAIL(SB200_EINVAL, "NULL segment handle");
  SB_CUDA(cudaSetDevice(seg->device));
  if (!batch || !totals) SB_FAIL(SB200_EINVAL, "NULL argument");
  return run_batch(seg, &batch->q, SB200_MODE_OR, batch, docs, nullptr, totals, n_out, stats);
}


int sb200_segment_attach_token_counts(sb200_segment* g, const uint64_t* counts, uint32_t max_doc) {
  if (!g || !counts) SB_FAIL(SB200_EINVAL, "NULL argument");
  if (max_doc != g->max_doc) SB_FAIL(SB200_EINVAL, "token counts for %u docs, the segment has %u", max_doc, g->max_doc);
  SB_CUDA(cudaSetDevice(g->device));
  g->has_tok = false;
  SB_TRY(g->tok_count.alloc(std::max<uint32_t>(max_doc, 1)));
  if (max_doc) SB_TRY(copy_in(g->tok_count.p, counts, (size_t)max_doc * 8, g->stream));
  SB_CUDA(cudaStreamSynchronize(g->stream));
  g->has_tok = true;
  return SB200_OK;
}

int sb200_pattern_docsets(sb200_segment* seg, const sb200_pattern_batch* batch, sb200_docset** out, sb200_pattern_stats* stats) {
  if (!seg) SB_FAIL(SB200_EINVAL, "NULL segment handle");
  SB_CUDA(cudaSetDevice(seg->device));
  return run_patterns(seg, batch, out, stats);
}

int sb200_docset_from_postings(sb200_segment* g, uint32_t term, sb200_docset** out) {
  if (!g || !out) SB_FAIL(SB200_EINVAL, "NULL argument");
  if (term != SB200_ABSENT_TERM && term >= g->n_terms) SB_FAIL(SB200_EINVAL, "term ordinal %u >= %u", term, g->n_terms);
  SB_CUDA(cudaSetDevice(g->device));
  // a one-TERM pattern takes the same path: its postings
  const uint8_t part = SB200_PART_TERM;
  sb200_pattern_batch b;
  memset(&b, 0, sizeof(b));
  b.n_patterns = 1; b.n_parts = 1; b.parts = &part; b.n_terms = 1; b.term_ords = &term;
  return run_patterns(g, &b, out, nullptr);
}

int sb200_docset_combine(int op, const sb200_docset* const* in, uint32_t n, sb200_docset** out) {
  if (!in || !out || n == 0) SB_FAIL(SB200_EINVAL, "NULL argument or no inputs");
  if (op != SB200_DOCSET_AND && op != SB200_DOCSET_OR) SB_FAIL(SB200_EINVAL, "op %d", op);
  for (uint32_t i = 0; i < n; i++) {
    if (!in[i]) SB_FAIL(SB200_EINVAL, "input %u is NULL", i);
    if (in[i]->max_doc != in[0]->max_doc || in[i]->device != in[0]->device)
      SB_FAIL(SB200_EINVAL, "input %u: max_doc %u on device %d, input 0: %u on %d", i, in[i]->max_doc, in[i]->device, in[0]->max_doc, in[0]->device);
  }
  SB_CUDA(cudaSetDevice(in[0]->device));
  sb200_docset* d = new (std::nothrow) sb200_docset;
  if (!d) SB_FAIL(SB200_ENOMEM, "docset: host allocation failed");
  d->device = in[0]->device; d->max_doc = in[0]->max_doc;
  const uint32_t nw = std::max<uint32_t>((in[0]->max_doc + 31) / 32, 1);
  std::vector<uint64_t> ptrs(n);
  for (uint32_t i = 0; i < n; i++) ptrs[i] = (uint64_t)(uintptr_t)in[i]->bits.p;
  DevBuf<uint64_t> dp;
  int rc = d->bits.alloc(nw);
  if (rc == SB200_OK) rc = dp.alloc(n);
  if (rc != SB200_OK) { delete d; return rc; }
  auto go = [&]() -> int {
    SB_CUDA(cudaMemcpy(dp.p, ptrs.data(), (size_t)n * 8, cudaMemcpyHostToDevice));
    SB_LAUNCH(k_docset_combine, div_up(nw, 256), 256, 0, 0, (const uint32_t* const*)dp.p, n, op == SB200_DOCSET_AND ? 0 : 1, d->bits.p, nw);
    SB_CHECK_LAUNCH();
    SB_CUDA(cudaDeviceSynchronize());
    return SB200_OK;
  };
  rc = go();
  if (rc != SB200_OK) { delete d; return rc; }
  *out = d;
  return SB200_OK;
}

int sb200_docset_count(const sb200_docset* ds, uint64_t* count) {
  if (!ds || !count) SB_FAIL(SB200_EINVAL, "NULL argument");
  SB_CUDA(cudaSetDevice(ds->device));
  DevBuf<unsigned long long> c;
  SB_TRY(c.alloc(1));
  SB_CUDA(cudaMemset(c.p, 0, 8));
  const uint32_t nw = (ds->max_doc + 31) / 32;
  if (nw) {
    SB_LAUNCH(k_docset_count, std::min<unsigned>(div_up(nw, 256), 1024u), 256, 0, 0, ds->bits.p, nw, c.p);
    SB_CHECK_LAUNCH();
  }
  unsigned long long h = 0;
  SB_CUDA(cudaMemcpy(&h, c.p, 8, cudaMemcpyDeviceToHost));
  *count = h;
  return SB200_OK;
}

// an inspection read-back: the bitmap crosses to the host and is expanded there
int sb200_docset_read(const sb200_docset* ds, uint32_t* docs, uint64_t cap, uint64_t* total) {
  if (!ds || !total || (cap && !docs)) SB_FAIL(SB200_EINVAL, "NULL argument");
  SB_CUDA(cudaSetDevice(ds->device));
  const uint32_t nw = (ds->max_doc + 31) / 32;
  std::vector<uint32_t> w(nw);
  if (nw) SB_CUDA(cudaMemcpy(w.data(), ds->bits.p, (size_t)nw * 4, cudaMemcpyDeviceToHost));
  std::vector<uint32_t> out;
  uint64_t n = 0;
  for (uint32_t i = 0; i < nw; i++)
    for (uint32_t x = w[i]; x; x &= x - 1) {
      if (n < cap) out.push_back(i * 32u + (uint32_t)__builtin_ctz(x));
      n++;
    }
  if (!out.empty()) SB_CUDA(cudaMemcpy(docs, out.data(), out.size() * 4, cudaMemcpyDefault));
  *total = n;
  return SB200_OK;
}

int sb200_docset_info(const sb200_docset* ds, uint32_t* max_doc, int* device) {
  if (!ds) SB_FAIL(SB200_EINVAL, "NULL docset handle");
  if (max_doc) *max_doc = ds->max_doc;
  if (device) *device = ds->device;
  return SB200_OK;
}

void sb200_docset_destroy(sb200_docset* ds) {
  if (!ds) return;
  cudaSetDevice(ds->device);
  delete ds;
}

int sb200_recall_plan_docs(const sb200_recall_plan_batch* plan, uint64_t* counts, uint32_t* docs, uint64_t cap, sb200_plan_stats* stats) {
  if (!plan || !counts || (cap && !docs)) SB_FAIL(SB200_EINVAL, "NULL argument");
  std::vector<uint32_t> h;
  auto emit = [&](uint32_t g0, uint32_t g1, const uint64_t* keys, const uint64_t*, const std::vector<uint64_t>& beg) -> int {
    const uint32_t n = g1 - g0;
    std::vector<uint64_t> c(n);
    for (uint32_t i = 0; i < n; i++) c[i] = beg[i + 1] - beg[i];
    SB_CUDA(cudaMemcpy(counts + g0, c.data(), (size_t)n * 8, cudaMemcpyDefault));
    if (!cap || beg[n] == 0) return SB200_OK;
    sb200_segment* g = plan->segments[0];
    DevBuf<uint32_t> d;
    SB_TRY(d.alloc(beg[n]));
    SB_LAUNCH(k_plan_docs, div_up(beg[n], 256), 256, 0, g->stream, keys, beg[n], d.p);
    SB_CHECK_LAUNCH();
    h.resize(beg[n]);
    SB_CUDA(cudaMemcpyAsync(h.data(), d.p, beg[n] * 4, cudaMemcpyDeviceToHost, g->stream));
    SB_CUDA(cudaStreamSynchronize(g->stream));
    for (uint32_t i = 0; i < n; i++) {
      const uint64_t c = std::min<uint64_t>(cap, beg[i + 1] - beg[i]);
      if (c) SB_CUDA(cudaMemcpy(docs + (size_t)(g0 + i) * cap, h.data() + beg[i], c * 4, cudaMemcpyDefault));
    }
    return SB200_OK;
  };
  return run_plan(plan, emit, stats);
}

int sb200_multi_signal_topk_batch_plan(const sb200_multi_signal_batch* batch, const sb200_recall_plan_batch* plan, const sb200_optic_batch* optic,
                                       uint32_t* docs, double* totals, uint32_t* n_out, sb200_bm25_stats* stats) {
  if (!plan) SB_FAIL(SB200_EINVAL, "NULL plan batch");
  return run_multi(batch, optic, docs, totals, n_out, stats, plan);
}

int sb200_multi_signal_webpages(const sb200_multi_signal_batch* batch, const sb200_optic_batch* optic, const sb200_webpage_batch* wb,
                                const sb200_webpage_out* out, sb200_webpage_stats* stats) {
  using namespace sb200;
  if (!batch || !batch->fields || !wb || !out) SB_FAIL(SB200_EINVAL, "NULL argument");
  if (wb->n_queries != batch->n_queries) SB_FAIL(SB200_EINVAL, "webpage batch has %u queries, signal batch %u", wb->n_queries, batch->n_queries);
  const uint32_t NF = batch->n_fields, nq = wb->n_queries, ndm = wb->n_docs_max;
  if (NF == 0 || NF > (uint32_t)M_MAX_FIELDS) SB_FAIL(SB200_ERANGE, "n_fields %u outside [1,%d]", NF, M_MAX_FIELDS);
  if ((uint64_t)nq * ndm > 0xFFFFFFFFull) SB_FAIL(SB200_ERANGE, "n_queries * n_docs_max = %llu above 2^32 - 1", (unsigned long long)nq * ndm);
  if (nq && (!wb->n_docs || (ndm && !wb->docs))) SB_FAIL(SB200_EINVAL, "NULL docs / n_docs");
  if (nq && ndm && (!out->values || !out->scores || !out->boosts || !out->min_slop)) SB_FAIL(SB200_EINVAL, "NULL output");
  const sb200_segment* g0 = batch->fields[0].seg;
  if (!g0) SB_FAIL(SB200_EINVAL, "field 0 has no segment");
  for (int f = 0; f < 2; f++) {
    const uint32_t x = wb->dist_field[f];
    if (x == SB200_WEBPAGE_NO_FIELD) continue;
    if (x >= NF) SB_FAIL(SB200_EINVAL, "distance field %d: field index %u >= %u", f, x, NF);
    if (!batch->fields[x].seg || !batch->fields[x].seg->has_pos) SB_FAIL(SB200_EINVAL, "distance field %d (field %u) has no positions attached", f, x);
  }
  if (wb->dist_field[0] != SB200_WEBPAGE_NO_FIELD && wb->dist_field[0] == wb->dist_field[1]) SB_FAIL(SB200_EINVAL, "both distance fields are field %u", wb->dist_field[0]);
  for (uint32_t q = 0; q < nq; q++) {
    if (wb->n_docs[q] > ndm) SB_FAIL(SB200_EINVAL, "query %u: n_docs %u > n_docs_max %u", q, wb->n_docs[q], ndm);
    for (uint32_t i = 0; i < wb->n_docs[q]; i++)
      if (wb->docs[(size_t)q * ndm + i] >= g0->max_doc) SB_FAIL(SB200_EINVAL, "query %u doc %u: %u >= max_doc %u", q, i, wb->docs[(size_t)q * ndm + i], g0->max_doc);
  }
  const WpCall wp{wb, out, stats};
  if (stats) memset(stats, 0, sizeof(*stats));
  return run_multi(batch, optic, nullptr, nullptr, nullptr, nullptr, nullptr, &wp);
}

int sb200_multi_signal_topk_batch_optic(const sb200_multi_signal_batch* batch, const sb200_optic_batch* optic, uint32_t* docs,
                                        double* totals, uint32_t* n_out, sb200_bm25_stats* stats) {
  if (!optic) SB_FAIL(SB200_EINVAL, "NULL optic batch");
  return run_multi(batch, optic, docs, totals, n_out, stats);
}

}  // extern "C"
