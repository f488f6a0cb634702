// bm25_multi.cuh -- Stract's recall-stage signals over SEVERAL text fields of one segment (SURVEY 8(f) rank 3).
//
// Reference: InitialSegmentScoreTweaker::score (core/src/ranking/initial.rs:79-93) over SignalComputeOrder::compute
// (core/src/ranking/computer/order.rs:17-135) with the TextFieldData methods bm25 / bm25f / coverage / idf_sum
// (core/src/ranking/computer/mod.rs:66-163), MultiBm25Weight (core/src/ranking/bm25.rs:47-107) and MultiBm25FWeight
// (core/src/ranking/bm25f.rs:79-181).
//
// Formulation: every (field, query term) pair is a "slot" with its own posting cursor; the union walk, the ownership
// rule (lowest slot containing a doc scores it), the per-block presence filters, the candidate buffer with its
// TopNComputer-style threshold, the doc-range work items and the merge pass are k_or3's (bm25_or3.cuh).  What is new
// is what happens once the term frequencies of a document are known for all slots: the document's fieldnorm id is
// fetched per field and a small "signal program" -- the ops of SignalComputeOrder in the reference's order, handed over
// by the host -- is evaluated in f64 exactly as the reference sums coefficient * score.
//   op kinds     0 bm25(field)   1 Bm25F = sum over the fields of bm25f   2 coverage(field)   3 idf_sum(field)
//                4 numeric column of the signal table
//   chain        n-gram groups (trigram, bigram, monogram of one field): score *= 0.4^hits, hits += score > 0
// Slots whose term is unknown to the segment stay in the query (SegmentPostings::empty(): they count in
// num_query_terms and keep their place in the f32 sums) with a zero doc_freq.
// Optic rule boosts (SignalComputer::boosts, computer/mod.rs:471-497): a rule's docset is a slot too (field | 0x80, its
// boost beside it), placed behind the text slots by the host.  Rule slots are probed, never enumerated on their own: a
// document owned by a rule slot is in no text slot and is skipped.  Matching rules add to `boost` or `downrank` in rule
// order and the total is multiplied by  downrank > boost ? 1/(1 + (downrank - boost)) : boost - downrank + 1.
// OPTIC = true (sb200_multi_signal_topk_batch_optic): rules are device docsets (bm25_pattern.cuh) instead of slots.  A
// candidate in the query's exclude bitmap or outside its require bitmap is dropped before scoring (the MustNot / Must filters
// of Discard and DiscardNonMatching); the rules' bits feed the same down / up sums in rule order and the same factor.
#pragma once

namespace sb200 {

constexpr int M_MAX_FIELDS = 6;
constexpr int M_MAX_OPS = 32;

struct MField {
  SegView S; const uint4* a128; const uint64_t* t_aoff;
  float cache[256];        // K1*(1-B+B*fieldnorm/avg) of the field (ranking/bm25.rs:29-45)
  float k1p1, coef;        // constants.k1 + 1.0; the field's signal coefficient as f32 (bm25f.rs:172)
  uint32_t n_terms, _pad;
};
struct MOp { uint32_t kind, field, chain, col; double coeff; };

struct MParams {
  const MField* fields; uint32_t n_fields, max_doc;
  const MOp* ops; uint32_t n_ops;
  const uint8_t* q_slot_field; const uint32_t* q_slot_term; const float* q_idf; const float* q_idf_f; const uint32_t* q_nslots;
  const double* q_boost;   // nullable: [nq][n_slots_max] boost of the rule slots
  const uint32_t* q_orig; uint32_t n_queries, n_slots_max, k, cap;
  uint32_t n_items; const uint32_t* item_q; const uint32_t* item_lo; const uint32_t* item_hi; const uint32_t* item_out;
  const double* sig; uint32_t n_cols;
  uint64_t* g_khi; uint32_t* g_klo;
  uint32_t* o_docs; double* o_totals; uint32_t* o_n; unsigned long long* counters;
  // optic docsets (k_sig_multi<TMAX, true>), per caller query index (q_orig): rules, boosts and the two filters
  const uint32_t* const* d_bits;   // [n_docsets] bitmaps
  const uint32_t* d_nrules; const uint32_t* d_rule; const double* d_boost; uint32_t d_max_rules;
  const uint32_t* d_exclude; const uint32_t* d_require;   // SB200_NO_DOCSET: none
};

__device__ __forceinline__ bool m_in(const uint32_t* bits, uint32_t d) { return (__ldg(bits + (d >> 5)) >> (d & 31u)) & 1u; }

template <int TMAX>
__host__ __device__ constexpr size_t m_warp_smem() { return (size_t)TMAX * 128 * 8 + (size_t)TMAX * 16 * 4 + (size_t)TMAX * sizeof(OTerm) + (size_t)TMAX * 8 + 48 * 4; }
template <int TMAX>
__host__ __device__ constexpr size_t m_cta_smem() { return M_MAX_FIELDS * 256 * 4 + M_MAX_OPS * sizeof(MOp) + WQ * m_warp_smem<TMAX>(); }

// What m_total reports besides the total: every op's (value before n-gram dampening, score after it) and every boost factor
// it multiplies the total with.  The top-k kernels pass MNoSink (ACTIVE = false: m_total compiles exactly as without a sink);
// k_wp_signals (bm25_webpage.cuh) keeps them.
struct MNoSink {
  static constexpr bool ACTIVE = false;
  __device__ __forceinline__ void op(const MOp&, uint32_t, double, double) {}
  __device__ __forceinline__ void boost(double) {}
};

// The per-candidate signal program of one document with the term frequencies of its T slots known (tf 0 = the slot does not
// hold it): the ops in order, the rule-slot boosts, then (OPTIC) the docset-rule boosts.  k_sig_multi, k_plan_recall
// (bm25_plan.cuh) and k_wp_signals (bm25_webpage.cuh) all call it, so a document gets the same f64 total whichever kernel
// found it.
template <int TMAX, bool OPTIC, class SINK>
__device__ __forceinline__ double m_total(const MParams& P, const MOp* s_ops, const float* s_cache, const uint32_t* s_nf, const uint32_t* s_fld,
                                          const float* s_wf, const OTerm* tc, uint32_t T, uint32_t q, uint32_t d, const uint32_t (&tf)[TMAX],
                                          uint32_t o_q, uint32_t o_nr, SINK& sink) {
  const uint32_t SM = P.n_slots_max;
  const double DAMP[3] = {1.0, 0.4, 0.4 * 0.4};   // NGRAM_DAMPENING.powi(hits) (order.rs:99,127)
  uint32_t fid[M_MAX_FIELDS];
#pragma unroll
  for (int f = 0; f < M_MAX_FIELDS; f++) fid[f] = ((uint32_t)f < P.n_fields) ? P.fields[f].S.fieldnorm[d] : 0u;
  double total = 0.0;
  int hits = 0;
  for (uint32_t o = 0; o < P.n_ops; o++) {
    const MOp op = s_ops[o];
    double sc = 0.0;
    if (op.kind == 4u) {
      sc = P.sig[(size_t)d * P.n_cols + op.col];
    } else if (op.kind == 1u) {
      // Bm25F: text_fields.values_mut().map(|f| f.bm25f(doc)).sum::<f64>() -- fields in EnumMap order, a field
      // without query terms is not in the map
#pragma unroll
      for (int f = 0; f < M_MAX_FIELDS; f++) {
        if ((uint32_t)f >= P.n_fields || s_nf[f] == 0) continue;
        const float norm = s_cache[f * 256 + fid[f]], k1p1 = P.fields[f].k1p1, coef = P.fields[f].coef;
        float b = 0.0f;
#pragma unroll
        for (int x = 0; x < TMAX; x++) if ((uint32_t)x < T && s_fld[x] == (uint32_t)f) {
          float part = 0.0f;
          if (tf[x]) { const float t = __fmul_rn((float)tf[x], coef); part = __fmul_rn(s_wf[x], __fdiv_rn(__fmul_rn(t, k1p1), __fadd_rn(t, norm))); }
          b = __fadd_rn(b, part);
        }
        sc = __dadd_rn(sc, (double)b);
      }
    } else if (s_nf[op.field] != 0) {
      const uint32_t f = op.field;
      if (op.kind == 0u) {
        const float norm = s_cache[f * 256 + fid[f]], k1p1 = P.fields[f].k1p1;
        float b = 0.0f;
#pragma unroll
        for (int x = 0; x < TMAX; x++) if ((uint32_t)x < T && s_fld[x] == f) {
          float part = 0.0f;
          if (tf[x]) { const float t = (float)tf[x]; part = __fmul_rn(tc[x].weight, __fdiv_rn(__fmul_rn(t, k1p1), __fadd_rn(t, norm))); }
          b = __fadd_rn(b, part);
        }
        sc = (double)b;
      } else if (op.kind == 2u) {
        double n = 0.0;
#pragma unroll
        for (int x = 0; x < TMAX; x++) if ((uint32_t)x < T && s_fld[x] == f) n = __dadd_rn(n, tf[x] ? 1.0 : 0.0);
        sc = __ddiv_rn(n, (double)s_nf[f]);
      } else if (op.kind == 3u) {
        float b = 0.0f;
#pragma unroll
        for (int x = 0; x < TMAX; x++) if ((uint32_t)x < T && s_fld[x] == f && tf[x]) b = __fadd_rn(b, tc[x].weight);
        sc = (double)b;
      }
    }
    double value = 0.0;
    if constexpr (SINK::ACTIVE) value = sc;
    if (op.chain) {
      if (op.chain == 1u) hits = 0;
      sc = __dmul_rn(sc, DAMP[hits > 2 ? 2 : hits]);
      if (sc > 0.0) hits++;
    }
    if constexpr (SINK::ACTIVE) sink.op(op, o, value, sc);
    total = __dadd_rn(total, __dmul_rn(op.coeff, sc));
  }
  if (P.q_boost) {   // SignalComputer::boosts
    double down = 0.0, up = 0.0;
#pragma unroll
    for (int x = 0; x < TMAX; x++) if ((uint32_t)x < T && (s_fld[x] & 0x80u) && tf[x]) {
      const double b = P.q_boost[(size_t)q * SM + x];
      if (b < 0.0) down = __dadd_rn(down, fabs(b)); else up = __dadd_rn(up, b);
    }
    const double factor = (down > up) ? __ddiv_rn(1.0, __dadd_rn(1.0, __dsub_rn(down, up))) : __dadd_rn(__dsub_rn(up, down), 1.0);
    if constexpr (SINK::ACTIVE) sink.boost(factor);
    total = __dmul_rn(total, factor);
  }
  if constexpr (OPTIC) {
    if (o_nr) {   // SignalComputer::boosts over the rule docsets, in rule order
      double down = 0.0, up = 0.0;
      for (uint32_t r = 0; r < o_nr; r++) {
        const size_t at = (size_t)o_q * P.d_max_rules + r;
        if (!m_in(P.d_bits[P.d_rule[at]], d)) continue;
        const double b = P.d_boost[at];
        if (b < 0.0) down = __dadd_rn(down, fabs(b)); else up = __dadd_rn(up, b);
      }
      const double factor = (down > up) ? __ddiv_rn(1.0, __dadd_rn(1.0, __dsub_rn(down, up))) : __dadd_rn(__dsub_rn(up, down), 1.0);
      if constexpr (SINK::ACTIVE) sink.boost(factor);
      total = __dmul_rn(total, factor);
    }
  }
  return total;
}

template <int TMAX, bool OPTIC = false>
__global__ void __launch_bounds__(WQ * 32) k_sig_multi(const MParams P) {
  SB_DYN_SMEM(smem_raw);
  float* s_cache = (float*)smem_raw;                                   // [M_MAX_FIELDS][256]
  MOp* s_ops = (MOp*)(smem_raw + M_MAX_FIELDS * 256 * 4);              // [M_MAX_OPS]
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char* wbase = smem_raw + M_MAX_FIELDS * 256 * 4 + M_MAX_OPS * sizeof(MOp) + warp * m_warp_smem<TMAX>();
  uint32_t* docs = (uint32_t*)wbase;                                   // [TMAX][128]
  uint32_t* tfs = docs + TMAX * 128;                                   // [TMAX][128]
  uint32_t* bloom = tfs + TMAX * 128;                                  // [TMAX][16]
  OTerm* tc = (OTerm*)(bloom + TMAX * 16);                             // [TMAX]
  float* s_wf = (float*)(tc + TMAX);                                   // [TMAX] bm25f idf
  uint32_t* s_fld = (uint32_t*)(s_wf + TMAX);                          // [TMAX] field of the slot (| 0x80: an optic rule's docset)
  uint32_t* s_misc = s_fld + TMAX;                                     // [48]
  uint32_t* s_rstart = s_misc;          // [TMAX + 1]
  uint32_t* s_pos = s_misc + 20;        // [TMAX]
  uint32_t* s_count = s_misc + 40;
  uint32_t* s_nf = s_misc + 41;         // [M_MAX_FIELDS] slots per field (num_query_terms)
  for (uint32_t i = threadIdx.x; i < P.n_fields * 256; i += WQ * 32) s_cache[i] = P.fields[i >> 8].cache[i & 255];
  for (uint32_t i = threadIdx.x; i < P.n_ops; i += WQ * 32) s_ops[i] = P.ops[i];
  __syncthreads();  // the only block barrier
  const uint32_t item = blockIdx.x * WQ + warp;
  if (item >= P.n_items) return;
  const uint32_t SM = P.n_slots_max;
  const uint32_t q = P.item_q ? P.item_q[item] : item;
  const uint32_t lo_doc = P.item_q ? P.item_lo[item] : 0u, hi_doc = P.item_q ? P.item_hi[item] : 0xFFFFFFFFu;
  const uint32_t oq = P.item_q ? P.item_out[item] : (P.q_orig ? P.q_orig[q] : q);
  const uint32_t T = min(P.q_nslots[q], (uint32_t)TMAX);
  uint64_t* khi = P.g_khi + (size_t)item * P.cap; uint32_t* klo = P.g_klo + (size_t)item * P.cap;
  const bool ranged = lo_doc > 0 || hi_doc != 0xFFFFFFFFu;
  const uint32_t* o_ex = nullptr; const uint32_t* o_rq = nullptr;
  uint32_t o_nr = 0, o_q = 0;
  if constexpr (OPTIC) {
    o_q = P.q_orig ? P.q_orig[q] : q;
    const uint32_t ex = P.d_exclude ? P.d_exclude[o_q] : SB200_NO_DOCSET, rq = P.d_require ? P.d_require[o_q] : SB200_NO_DOCSET;
    if (ex != SB200_NO_DOCSET) o_ex = P.d_bits[ex];
    if (rq != SB200_NO_DOCSET) o_rq = P.d_bits[rq];
    o_nr = P.d_nrules ? P.d_nrules[o_q] : 0u;
  }

  // ---- cursors: lane t owns slot t
  uint32_t my_pos = 0, my_len = 0, my_last = 0, my_cur = 0, my_prev = 0;
  bool my_done = true, my_tail_done = false;
  unsigned long long budget = 64;
  if (lane < M_MAX_FIELDS) s_nf[lane] = 0;
  __syncwarp();
  if (lane < T) {
    OTerm c;
    memset(&c, 0, sizeof(c));
    const uint32_t fr = P.q_slot_field[(size_t)q * SM + lane];
    const uint32_t f = fr & 0x7Fu;
    const uint32_t ord = P.q_slot_term[(size_t)q * SM + lane];
    const MField& F = P.fields[f];
    if (ord != SB200_NO_TERM && ord < F.n_terms) {
      c.first = F.S.t_first[ord]; c.df = F.S.t_df[ord]; c.nfull = c.df >> 7;
      c.adata = F.t_aoff[ord]; c.end_off = F.S.t_end_off[ord];
      c.tail_off = F.S.t_data_off[ord] + F.S.b_off[c.first + c.nfull];
    }
    c.weight = P.q_idf[(size_t)q * SM + lane];
    tc[lane] = c; s_wf[lane] = P.q_idf_f[(size_t)q * SM + lane]; s_fld[lane] = fr;
    if (!(fr & 0x80u)) atomicAdd(s_nf + f, 1u);   // num_query_terms counts text slots only
    my_done = (c.df == 0);
    budget = 4ull * (c.nfull + 2);
  }
  for (uint32_t i = lane; i < TMAX * 16; i += 32) bloom[i] = 0;
  if (lane == 0) *s_count = 0;
  for (int o = 16; o; o >>= 1) budget += __shfl_xor_sync(0xffffffffu, budget, o);
  __syncwarp();
  if (lo_doc > 0) {  // start every cursor at the first block that can hold a doc >= lo
    for (uint32_t s = 0; s < T; s++) {
      const OTerm& c = tc[s];
      if (c.nfull == 0) continue;
      const uint32_t j = o3_dir_search(P.fields[s_fld[s] & 0x7Fu].S.b_last + c.first, 0, c.nfull, lo_doc, lane);
      if (lane == s && j > 0) { my_cur = j; my_prev = P.fields[s_fld[s] & 0x7Fu].S.b_last[c.first + j - 1]; }
    }
  }
  bool thr_on = false; uint64_t thr_hi = 0; uint32_t thr_lo = 0;   // warp-uniform
  unsigned long long my_docs = 0, my_blocks = 0;
  bool watchdog = false, bad_doc = false;

  while (T > 0) {
    if (budget-- == 0) { watchdog = true; break; }
    // ---- (1) refill every exhausted cursor
    for (;;) {
      unsigned need = __ballot_sync(0xffffffffu, lane < T && !my_done && my_pos >= my_len);
      if (!need) break;
      while (need) {
        const int s = __ffs(need) - 1; need &= need - 1;
        const uint32_t cur = __shfl_sync(0xffffffffu, my_cur, s), prev = __shfl_sync(0xffffffffu, my_prev, s);
        const bool tdone = __shfl_sync(0xffffffffu, (int)my_tail_done, s) != 0;
        const OTerm c = tc[s];
        const bool more = (cur < c.nfull) || (cur == c.nfull && !tdone && (c.df & 127u));
        if (!more) {
          if (lane == (uint32_t)s) my_done = true;
          __syncwarp();
          if (lane < 16) bloom[s * 16 + lane] = 0;
          __syncwarp();
          continue;
        }
        uint32_t last;
        const MField& F = P.fields[s_fld[s] & 0x7Fu];
        const uint32_t n = o3_decode(F.S, F.a128, c, cur, prev, docs + s * 128, tfs + s * 128, bloom + s * 16, lane, last);
        my_blocks++;
        if (lane == (uint32_t)s) {
          my_len = n; my_pos = 0; my_last = last; my_prev = last; my_cur = cur + 1;
          if (cur >= c.nfull) my_tail_done = true;
          if (ranged) {
            const uint32_t p = lower_bound128(docs + s * 128, lo_doc);
            my_pos = min(p, n);
            if (my_pos < my_len && docs[s * 128 + my_pos] >= hi_doc) my_done = true;
          }
        }
      }
      if (budget-- == 0) { watchdog = true; break; }
    }
    if (watchdog) break;
    // ---- (2) bound
    const bool active = lane < T && !my_done;
    if (!__any_sync(0xffffffffu, active)) break;
    uint32_t bound = __reduce_min_sync(0xffffffffu, active ? my_last : 0xFFFFFFFFu);
    if (ranged && bound >= hi_doc) bound = hi_doc - 1u;
    // ---- (3) this round's slice of every slot
    uint32_t rhi = my_pos;
    if (active) rhi = min(lower_bound128(docs + lane * 128, bound + 1u), my_len);
    const uint32_t cnt = rhi - my_pos;
    const uint32_t incl = warp_scan_incl(cnt, lane);
    const uint32_t R = __shfl_sync(0xffffffffu, incl, 31);
    __syncwarp();
    if (lane <= T) s_rstart[lane] = incl - cnt;
    if (lane < T) s_pos[lane] = my_pos;
    const uint32_t have = *s_count;
    __syncwarp();
    if (have + R > P.cap) {
      w_sort_prefix_desc(khi, klo, have, P.cap, lane);
      const uint32_t c = min(have, P.k);
      if (c == P.k) { thr_on = true; thr_hi = khi[P.k - 1]; thr_lo = klo[P.k - 1]; }
      __syncwarp();
      if (lane == 0) *s_count = c;
      __syncwarp();
    }
    // ---- (4) score
    for (uint32_t e = lane; e < R; e += 32) {
      uint32_t i = 0;
#pragma unroll
      for (int x = 1; x < TMAX; x++) if ((uint32_t)x < T && e >= s_rstart[x]) i = x;
      const uint32_t pj = s_pos[i] + (e - s_rstart[i]);
      const uint32_t d = docs[i * 128 + pj];
      if (d >= P.max_doc) { bad_doc = true; continue; }
      const uint32_t bw = (d >> 5) & 15u, bb = 1u << (d & 31u);
      uint32_t tf[TMAX];
      bool owner = true;
#pragma unroll
      for (int x = 0; x < TMAX; x++) {
        tf[x] = 0;
        if ((uint32_t)x >= T || !owner) continue;
        if ((uint32_t)x == i) { tf[x] = tfs[i * 128 + pj]; continue; }
        if (!(bloom[x * 16 + bw] & bb)) continue;
        const uint32_t jj = lower_bound128(docs + x * 128, d);
        if (jj < 128u && docs[x * 128 + jj] == d) {
          if ((uint32_t)x < i) owner = false;
          else tf[x] = tfs[x * 128 + jj];
        }
      }
      if (!owner) continue;
      if (s_fld[i] & 0x80u) continue;   // only rule docsets hold this doc: not a candidate
      if constexpr (OPTIC) {
        if (o_ex && m_in(o_ex, d)) continue;    // Discard rules, blocked hosts
        if (o_rq && !m_in(o_rq, d)) continue;   // DiscardNonMatching
      }
      my_docs++;
      MNoSink none;
      const double total = m_total<TMAX, OPTIC>(P, s_ops, s_cache, s_nf, s_fld, s_wf, tc, T, q, d, tf, o_q, o_nr, none);
      const uint64_t kh = ord_f64(total);
      const uint32_t kl = ~d;
      if (thr_on && !key_gt(kh, kl, thr_hi, thr_lo)) continue;
      const uint32_t at = atomicAdd(s_count, 1u);
      khi[at] = kh; klo[at] = kl;
    }
    // ---- (5) consume the slice
    if (active) {
      my_pos = rhi;
      if (ranged && my_pos < my_len && docs[lane * 128 + my_pos] >= hi_doc) my_done = true;
    }
    __syncwarp();
  }
  __threadfence_block();
  __syncwarp();
  w_sort_prefix_desc(khi, klo, *s_count, P.cap, lane);
  const uint32_t n = min(*s_count, P.k);
  for (uint32_t i = lane; i < n; i += 32) {
    P.o_docs[(size_t)oq * P.k + i] = ~klo[i];
    P.o_totals[(size_t)oq * P.k + i] = unord_f64(khi[i]);
  }
  if (lane == 0) P.o_n[oq] = n;
  for (int o = 16; o; o >>= 1) my_docs += __shfl_down_sync(0xffffffffu, my_docs, o);
  if (__any_sync(0xffffffffu, bad_doc)) watchdog = true;
  if (lane == 0) {
    if (my_docs) atomicAdd(P.counters + 0, my_docs);
    if (my_blocks) atomicAdd(P.counters + 1, my_blocks);
    if (watchdog) atomicAdd(P.counters + 2, 1ull);
  }
}

}  // namespace sb200
