// bm25_wand.cuh -- tantivy's Block-Max WAND replayed step by step on the device (SB200_MODE_OR_WAND).
//
// Why it exists: for a Should-only query with >= 3 terms tantivy sums the term scores of a document in the order its
// scorer array happens to have when the document becomes the pivot (`scorers[..pivot_len].map(score).sum()`,
// crates/tantivy/src/query/boolean_query/block_wand.rs:195-198), and that order is a function of the whole pruning history
// (restore_ordering :88-97, swap_remove in align_scorers :113-116 and advance_all_scorers_on_pivot :139-146, the stable
// re-sort :147).  f32 addition is not associative, so the exhaustive union kernel -- which sums in query order -- can
// differ from the reference in the last ulp of a score and thereby in the order of two near-tied documents (measured on
// C5-style 5-term queries, top-1000: 0.1 % of the queries change their doc order, 18 % some score bit).  The only way to
// reproduce a history is to walk it: this kernel is block_wand itself, one warp per query, with the reference's
// TermScorer / SkipReader / TopNComputer state machines:
//   find_pivot_doc :16-43, block_max_was_too_low_advance_one_scorer :49-83, restore_ordering :88-97,
//   align_scorers :104-123, advance_all_scorers_on_pivot :128-148, block_wand :153-214,
//   SkipReader::seek/advance (postings/skip.rs:234-281), BlockSegmentPostings::block_max_score
//   (postings/block_segment_postings.rs:147-184), SegmentPostings::seek/advance (postings/segment_postings.rs:157-193),
//   TopNComputer::push/truncate_top_n (collector/top_score_collector.rs:501-554).
// All control state is warp-uniform and PRIVATE: every lane runs the same scalar program on its own copy of the scorer
// structs (thread-local arrays), so no lane ever depends on another lane's progress; the lanes cooperate only where the
// data is wide -- decoding a 128-doc block into shared memory, a block maximum, sorting the candidate buffer.  It is one
// to two orders of magnitude slower than the exhaustive kernel -- it is the reference's algorithm, with the reference's
// pruning -- and is selected explicitly when score bits must match.
#pragma once

namespace sb200 {

constexpr int WD_MAXT = SB200_MAX_QUERY_TERMS;
constexpr int WD_WARPS = 4;

struct WScorer {   // one TermScorer: weights, skip reader and block cursor (warp-uniform)
  uint64_t adata, tail_off, end_off;
  uint32_t first, nfull, df;
  float weight, max_sc;
  uint32_t blk;        // skip reader position: block index; blk == nfull is the vint tail, blk > nfull the empty block behind it
  uint32_t last;       // skip.last_doc_in_block
  uint32_t loaded;     // block index whose docs / tfs are in shared memory (0xFFFFFFFF: none)
  uint32_t cur, len;   // cursor inside the loaded block, number of postings in it
  uint32_t has_bm; float bm;
  uint32_t _pad;
};

struct WandParams {
  SegView S; const uint16_t* b_bw;     // per block: block-wand (fieldnorm id | tf << 8) of the skip entry
  const uint4* a128; const uint64_t* t_aoff;
  const uint32_t* q_terms; const uint32_t* q_nterms; const float* q_weights; const float* cache; const uint32_t* q_orig;
  uint32_t n_queries, n_terms_max, k, cap;
  uint64_t* g_khi; uint32_t* g_klo;
  uint32_t* o_docs; float* o_scores; uint32_t* o_n; unsigned long long* counters;
};

__device__ __forceinline__ float wd_score(float weight, const float* cache, uint32_t id, uint32_t tf) {
  const float t = (float)tf;
  return __fmul_rn(weight, __fdiv_rn(t, __fadd_rn(t, cache[id])));   // Bm25Weight::score, bm25.rs:182-196
}
__device__ __forceinline__ uint32_t wd_last_of(const WandParams& P, const WScorer& s, uint32_t blk) {
  return blk < s.nfull ? P.S.b_last[s.first + blk] : TERMINATED;
}
// SkipReader::seek: move to the first block whose last doc >= target; true if it moved
__device__ __forceinline__ bool wd_skip_seek(const WandParams& P, WScorer& s, uint32_t target) {
  if (s.last >= target) return false;
  do { s.blk++; s.last = wd_last_of(P, s, s.blk); } while (s.last < target);
  return true;
}
// BlockSegmentPostings::load_block for the skip reader's current block (every lane calls it)
__device__ void wd_load(const WandParams& P, WScorer& s, uint32_t* docs, uint32_t* tfs, uint32_t* scratch, uint32_t lane) {
  if (s.loaded == s.blk) return;
  if (s.blk < s.nfull || (s.blk == s.nfull && (s.df & 127u))) {
    OTerm c;
    c.adata = s.adata; c.tail_off = s.tail_off; c.end_off = s.end_off; c.first = s.first; c.nfull = s.nfull; c.df = s.df; c.weight = 0.f;
    const uint32_t prev = s.blk ? P.S.b_last[s.first + s.blk - 1] : 0u;
    uint32_t last;
    s.len = o3_decode(P.S, P.a128, c, s.blk, prev, docs, tfs, scratch, lane, last);
  } else {   // nothing left: an empty block, every doc TERMINATED (skip.rs:262-267, block_segment_postings.rs:334-349)
    __syncwarp();
    for (uint32_t i = lane; i < 128; i += 32) { docs[i] = TERMINATED; tfs[i] = 0; }
    __syncwarp();
    s.len = 0;
  }
  s.loaded = s.blk;
}
__device__ __forceinline__ void wd_shallow_seek(const WandParams& P, WScorer& s, uint32_t target) {
  if (wd_skip_seek(P, s, target)) { s.has_bm = 0; s.loaded = 0xFFFFFFFFu; }   // the decoded block no longer belongs to the skip position
}
__device__ uint32_t wd_seek(const WandParams& P, WScorer& s, uint32_t* docs, uint32_t* tfs, uint32_t* scratch, uint32_t target, uint32_t lane) {
  if (docs[s.cur] >= target) return docs[s.cur];   // SegmentPostings::seek looks at the decoded buffer as it is, stale or not
  wd_shallow_seek(P, s, target);
  wd_load(P, s, docs, tfs, scratch, lane);
  s.cur = min(lower_bound128(docs, target), 127u);
  return docs[s.cur];
}
__device__ uint32_t wd_advance(const WandParams& P, WScorer& s, uint32_t* docs, uint32_t* tfs, uint32_t* scratch, uint32_t lane) {
  if (s.cur == 127u) {
    s.cur = 0; s.blk++; s.last = wd_last_of(P, s, s.blk); s.has_bm = 0; s.loaded = 0xFFFFFFFFu;
    wd_load(P, s, docs, tfs, scratch, lane);
  } else s.cur++;
  return docs[s.cur];
}
__device__ float wd_block_max(const WandParams& P, WScorer& s, const uint32_t* docs, const uint32_t* tfs, const float* cache, uint32_t lane) {
  if (s.has_bm) return s.bm;
  if (s.blk < s.nfull) {
    const uint32_t bw = P.b_bw[s.first + s.blk];
    const uint32_t tf = (bw >> 8) == 255u ? 0xFFFFFFFFu : (bw >> 8);
    s.bm = wd_score(s.weight, cache, bw & 0xFFu, tf); s.has_bm = 1;
    return s.bm;
  }
  if (s.loaded == s.blk) {   // the vint tail, decoded: the maximum over its postings (0 for an empty block)
    float best = 0.0f;
    for (uint32_t i = lane; i < s.len; i += 32) best = fmaxf(best, wd_score(s.weight, cache, P.S.fieldnorm[docs[i]], tfs[i]));
    for (int o = 16; o; o >>= 1) best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, o));
    s.bm = best; s.has_bm = 1;
    return best;
  }
  return s.max_sc;
}

__global__ void __launch_bounds__(WD_WARPS * 32) k_wand(const WandParams P) {
  __shared__ float cache[256];
  __shared__ __align__(16) uint32_t s_docs[WD_WARPS][WD_MAXT * 128];
  __shared__ __align__(16) uint32_t s_tfs[WD_WARPS][WD_MAXT * 128];
  __shared__ uint32_t s_scratch[WD_WARPS][16];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (uint32_t i = threadIdx.x; i < 256; i += WD_WARPS * 32) cache[i] = P.cache[i];
  __syncthreads();
  const uint32_t q = blockIdx.x * WD_WARPS + warp;
  if (q >= P.n_queries) return;
  WScorer sc[WD_MAXT];        // thread-local: identical in every lane
  uint32_t ord[WD_MAXT];      // the scorer array of block_wand, as indices into sc
  uint32_t* scratch = s_scratch[warp];
#define WD_DOCS(i) (s_docs[warp] + (i) * 128)
#define WD_TFS(i) (s_tfs[warp] + (i) * 128)
#define WD_DOC(i) (WD_DOCS(i)[sc[i].cur])
  const uint32_t TM = P.n_terms_max;
  uint32_t n = min(P.q_nterms[q], (uint32_t)WD_MAXT);
  uint64_t* khi = P.g_khi + (size_t)q * P.cap; uint32_t* klo = P.g_klo + (size_t)q * P.cap;
  const uint32_t oq = P.q_orig ? P.q_orig[q] : q;
  // ---- TermScorers (term_scorer.rs) positioned on their first doc
  for (uint32_t i = 0; i < n; i++) {
    WScorer s;
    const uint32_t t = P.q_terms[(size_t)q * TM + i];
    s.first = P.S.t_first[t]; s.df = P.S.t_df[t]; s.nfull = s.df >> 7;
    s.adata = P.t_aoff[t]; s.end_off = P.S.t_end_off[t];
    s.tail_off = P.S.t_data_off[t] + P.S.b_off[s.first + s.nfull];
    s.weight = P.q_weights[(size_t)q * TM + i];
    s.max_sc = wd_score(s.weight, cache, 255u, 2013265944u);   // Bm25Weight::max_score, bm25.rs:178-180
    s.blk = 0; s.last = s.nfull ? P.S.b_last[s.first] : TERMINATED; s.loaded = 0xFFFFFFFFu; s.cur = 0; s.len = 0; s.has_bm = 0; s.bm = 0.f; s._pad = 0;
    sc[i] = s;
    wd_load(P, sc[i], WD_DOCS(i), WD_TFS(i), scratch, lane);
    ord[i] = i;
  }
  // scorers.sort_by_key(doc): stable insertion sort
  for (uint32_t i = 1; i < n; i++) {
    const uint32_t x = ord[i]; const uint32_t dx = WD_DOC(x);
    uint32_t j = i;
    while (j > 0 && WD_DOC(ord[j - 1]) > dx) { ord[j] = ord[j - 1]; j--; }
    ord[j] = x;
  }
  // ---- TopNComputer
  const uint32_t top_n = P.k, tcap = 2u * P.k;
  uint32_t count = 0; bool has_thr = false; float thr = 0.f;
  float threshold = -3.4028235e38f;
  unsigned long long n_scored = 0, n_blocks = 0;
  unsigned long long guard = 64ull;
  for (uint32_t i = 0; i < n; i++) guard += 600ull * (sc[i].df + 256ull);   // a broken build fails instead of spinning
  bool watchdog = false;
  // TopNComputer::push, then the collector's new threshold (the callback of both walks)
  auto push = [&](float score, uint32_t doc) {
    if (!(score > threshold)) return;
    if (!(has_thr && score < thr)) {
      if (count == tcap) {
        w_sort_prefix_desc(khi, klo, count, P.cap, lane);
        thr = unord_f32((uint32_t)(khi[top_n] >> 32)); has_thr = true; count = top_n;
        __syncwarp();
      }
      if (lane == 0) { khi[count] = (uint64_t)ord_f32(score) << 32; klo[count] = ~doc; }
      count++;
      __syncwarp();
    }
    threshold = has_thr ? thr : -3.4028235e38f;
  };

  if (n == 1) {
    // A one-clause query is not block_wand in the reference: the TermWeight runs block_wand_single_scorer
    // (term_weight.rs:81-90, block_wand.rs:222-261).  It has no max_score cut-off, skips a block while its block max is
    // below (not at) the threshold, and leaves a scored block with shallow_seek(last + 1), so the next block is not
    // loaded: a VInt tail it has not loaded is bounded by max_score (block_segment_postings.rs:147-184), which is no
    // bound on a large tf in a short document.  This walk restates it step by step.
    WScorer& s = sc[0];
    uint32_t* docs = WD_DOCS(0); uint32_t* tfs = WD_TFS(0);
    uint32_t doc = docs[s.cur];
    for (;;) {
      if (guard-- == 0) { watchdog = true; break; }
      bool done = false;
      while (wd_block_max(P, s, docs, tfs, cache, lane) < threshold) {
        if (s.last == TERMINATED) { done = true; break; }
        doc = s.last + 1; wd_shallow_seek(P, s, doc); n_blocks++;
      }
      if (done) break;
      doc = wd_seek(P, s, docs, tfs, scratch, doc, lane);
      if (doc == TERMINATED) break;
      bool ret = false;
      for (;;) {
        push(wd_score(s.weight, cache, P.S.fieldnorm[doc], tfs[s.cur]), doc); n_scored++;
        if (doc == s.last) break;
        doc = wd_advance(P, s, docs, tfs, scratch, lane);
        if (doc == TERMINATED) { ret = true; break; }
      }
      if (ret) break;
      doc += 1; wd_shallow_seek(P, s, doc);
    }
    n = 0;   // the block_wand loop below has nothing to do
  }

#define WD_RESTORE(ordinal)                                                              \
  do {                                                                                    \
    const uint32_t _d = WD_DOC(ord[ordinal]);                                             \
    for (uint32_t _i = (ordinal) + 1; _i < n; _i++) {                                     \
      if (WD_DOC(ord[_i]) >= _d) break;                                                   \
      const uint32_t _t = ord[_i]; ord[_i] = ord[_i - 1]; ord[_i - 1] = _t;              \
    }                                                                                     \
  } while (0)

  for (;;) {
    if (guard-- == 0) { watchdog = true; break; }
    // find_pivot_doc
    float ms = 0.0f; uint32_t before = 0, pivot = TERMINATED;
    while (before < n) { ms = __fadd_rn(ms, sc[ord[before]].max_sc); if (ms > threshold) { pivot = WD_DOC(ord[before]); break; } before++; }
    if (pivot == TERMINATED) break;
    uint32_t plen = before + 1;
    while (plen < n && WD_DOC(ord[plen]) == pivot) plen++;
    float ub = 0.0f;
    for (uint32_t i = 0; i < plen; i++) {
      const uint32_t x = ord[i];
      wd_shallow_seek(P, sc[x], pivot);
      ub = __fadd_rn(ub, wd_block_max(P, sc[x], WD_DOCS(x), WD_TFS(x), cache, lane));
    }
    if (ub <= threshold) {   // block_max_was_too_low_advance_one_scorer
      uint32_t to_seek = plen - 1; float gmax = sc[ord[to_seek]].max_sc; uint32_t after = sc[ord[to_seek]].last;
      for (uint32_t i = plen - 1; i-- > 0;) {
        const WScorer& s = sc[ord[i]];
        if (s.last <= after) after = s.last;
        if (s.max_sc > gmax) { gmax = s.max_sc; to_seek = i; }
      }
      if (after != TERMINATED) after += 1;
      for (uint32_t i = plen; i < n; i++) { const uint32_t d = WD_DOC(ord[i]); if (d <= after) after = d; }
      const uint32_t x = ord[to_seek];
      wd_seek(P, sc[x], WD_DOCS(x), WD_TFS(x), scratch, after, lane); n_blocks++;
      WD_RESTORE(to_seek);
      continue;
    }
    // align_scorers
    bool aligned = true;
    for (uint32_t i = before; i-- > 0;) {
      const uint32_t x = ord[i];
      const uint32_t nd = wd_seek(P, sc[x], WD_DOCS(x), WD_TFS(x), scratch, pivot, lane);
      if (nd != pivot) {
        if (nd == TERMINATED) { ord[i] = ord[n - 1]; n--; }   // swap_remove
        if (i < n) WD_RESTORE(i);
        aligned = false; break;
      }
    }
    if (!aligned) continue;
    // all of scorers[..pivot_len] sit on the pivot: sum their scores in array order
    float score = 0.0f;
    {
      const uint32_t id = P.S.fieldnorm[pivot];
      for (uint32_t i = 0; i < plen; i++) { const uint32_t x = ord[i]; score = __fadd_rn(score, wd_score(sc[x].weight, cache, id, WD_TFS(x)[sc[x].cur])); }
    }
    n_scored++;
    push(score, pivot);
    // advance_all_scorers_on_pivot
    for (uint32_t i = 0; i < plen; i++) { const uint32_t x = ord[i]; wd_advance(P, sc[x], WD_DOCS(x), WD_TFS(x), scratch, lane); }
    for (uint32_t i = 0; i != n;) { if (WD_DOC(ord[i]) == TERMINATED) { ord[i] = ord[n - 1]; n--; } else i++; }
    for (uint32_t i = 1; i < n; i++) {   // sort_by_key(doc), stable
      const uint32_t x = ord[i]; const uint32_t dx = WD_DOC(x);
      uint32_t j = i;
      while (j > 0 && WD_DOC(ord[j - 1]) > dx) { ord[j] = ord[j - 1]; j--; }
      ord[j] = x;
    }
  }
  // into_sorted_vec
  __syncwarp();
  w_sort_prefix_desc(khi, klo, count, P.cap, lane);
  const uint32_t m = min(count, top_n);
  for (uint32_t i = lane; i < m; i += 32) {
    P.o_docs[(size_t)oq * P.k + i] = ~klo[i];
    P.o_scores[(size_t)oq * P.k + i] = unord_f32((uint32_t)(khi[i] >> 32));
  }
  if (lane == 0) {
    P.o_n[oq] = m;
    atomicAdd(P.counters + 0, n_scored);
    atomicAdd(P.counters + 1, n_blocks);
    if (watchdog) atomicAdd(P.counters + 2, 1ull);
  }
#undef WD_RESTORE
#undef WD_DOC
#undef WD_TFS
#undef WD_DOCS
}

}  // namespace sb200
