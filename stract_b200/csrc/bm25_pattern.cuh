// bm25_pattern.cuh -- optic pattern rules as device docsets: Stract's PatternQuery (core/src/query/pattern_query/) evaluated
// to one bit per document, and the AND / OR of such bitmaps that optic rules are made of (core/src/query/optic.rs:104-169).
//
// A docset is ceil(max_doc / 32) u32 words; bit d of word d >> 5 is document d, bits at or past max_doc are 0.  A rule's
// docset is only ever asked "is doc d in it?" (SignalComputer::boosts, the Discard / DiscardNonMatching filters of the recall
// query), so the bitmap is the exact representation and word-wise AND / OR the exact composition.
//
// PatternWeight::pattern_scorer (weight.rs:121-226) picks the branch from the tokenised parts alone; the host does the same:
//   no parts                              -> empty
//   no terms, a wildcard                  -> every document (AllScorer)                          k_docset_all
//   no terms, anchors only                -> token count (unwrap_or_default) == 0 (EmptyFieldScorer)   k_docset_empty_field
//   a term the segment lacks              -> empty (read_postings -> None)
//   one term and nothing else             -> its postings (the term_freq > 0 shortcut)           k_docset_postings
//   otherwise                             -> NormalPatternScorer:
//     k_phrase_cand    (bm25_phrase.cuh) the AND of the terms, with every term's tf and position offset per candidate
//     k_pattern_verify one warp per candidate: the terms' positions into shared memory (global scratch for long lists), then
//                      left = positions of term 0 and, per later term, left = intersection_with_slop(left, right, slop) with
//                      slop 1 (u32::MAX after a wildcard).  That function (scorer.rs:371-409) returns exactly
//                        { r in right : some l in left with r -| slop <= l <= r }      (-| saturating)
//                      so every lane binary-searches its own r for the largest l <= r, and the filtered right is compacted in
//                      place (it is a subset of right: no growth, one fallback pass).  Anchors: index 0 checks the first
//                      position of term 0, the last index checks the last position of the last term's raw list against
//                      (num_tokens - 1) as u32; anchors elsewhere are ignored (scorer.rs:313-333).
//                      A match sets its bit with atomicOr: the result is a set, the same for any schedule.
// FastSiteDomainPatternWeight (pattern_query/mod.rs:61-92) is one posting list: sb200_docset_from_postings.
#pragma once

namespace sb200 {

constexpr int PT_WARPS = 4;                  // candidates (warps) per CTA of k_pattern_verify
constexpr uint32_t PT_SMEM_WORDS = 1536;     // per-warp position buffer in shared memory

// every doc of term q_terms[u.q * n_terms_max] (slot 0 of the unit's row) into the bitmap out[u.q]
__global__ void __launch_bounds__(A3_WARPS * 32) k_docset_postings(const A3Params P, uint32_t* const* out) {
  __shared__ __align__(16) uint32_t s_docs[A3_WARPS][128];
  __shared__ __align__(16) uint32_t s_tfs[A3_WARPS][128];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t u = blockIdx.x * A3_WARPS + warp;
  if (u >= P.n_units) return;
  const AUnit U = P.units[u];
  const A3Term t = a3_load_term(P, U.q, 0);
  uint32_t* bits = out[U.q];
  bool bad = false;
  for (uint32_t blk = U.blk_lo; blk < U.blk_hi; blk++) {
    uint32_t d[4], n = 128;
    if (blk < t.nfull) {
      A3Blk B;
      const uint4 v = a3_decode_docs(P, t, blk, lane, B);
      d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
    } else {
      n = a3_decode_tail(P, t, s_docs[warp], s_tfs[warp], lane);
      const uint4 v = ((const uint4*)s_docs[warp])[lane];
      d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
      __syncwarp();
    }
#pragma unroll
    for (int b = 0; b < 4; b++) if (lane * 4 + b < n) {
      if (d[b] < P.S.max_doc) atomicOr(bits + (d[b] >> 5), 1u << (d[b] & 31u));
      else bad = true;
    }
  }
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicAdd(P.counters + 2, 1ull);
}

// AllScorer: every document below max_doc
__global__ void k_docset_all(uint32_t* bits, uint32_t max_doc) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t nw = (max_doc + 31) >> 5;
  if (w >= nw) return;
  const uint32_t lo = w << 5;
  bits[w] = (max_doc - lo >= 32) ? 0xFFFFFFFFu : ((1u << (max_doc - lo)) - 1u);
}

// EmptyFieldScorer: the documents whose token count is 0 (a missing value is passed as 0: unwrap_or_default)
__global__ void k_docset_empty_field(const uint64_t* __restrict__ counts, uint32_t* bits, uint32_t max_doc) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t nw = (max_doc + 31) >> 5;
  if (w >= nw) return;
  uint32_t m = 0;
  for (uint32_t b = 0; b < 32; b++) {
    const uint32_t d = (w << 5) + b;
    if (d < max_doc && __ldg(counts + d) == 0) m |= 1u << b;
  }
  bits[w] = m;
}

// word-wise AND (op 0) / OR (op 1) of n bitmaps
__global__ void k_docset_combine(const uint32_t* const* in, uint32_t n, int op, uint32_t* out, uint32_t n_words) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n_words) return;
  uint32_t v = __ldg(in[0] + w);
  for (uint32_t i = 1; i < n; i++) { const uint32_t x = __ldg(in[i] + w); v = op == 0 ? (v & x) : (v | x); }
  out[w] = v;
}

__global__ void k_docset_count(const uint32_t* __restrict__ bits, uint32_t n_words, unsigned long long* out) {
  uint32_t c = 0;
  for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += gridDim.x * blockDim.x) c += __popc(__ldg(bits + w));
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, (unsigned long long)c);
}

// ------------------------------------------------------------------ verification ------------------------------------------
struct PtParams {
  PosView V;
  const uint32_t* q_terms;     // per query slot, [slot * nt + c]: the term of candidate record column c (docset order)
  const uint32_t* q_col;       // per query slot, [slot * nt + j]: the record column of pattern term j
  const uint8_t* q_parts;      // per query slot, [slot * np + i]
  const uint32_t* q_nparts;    // per query slot
  const uint32_t* q_nterms;    // per query slot
  uint32_t nt, np;
  const uint64_t* token_counts;   // NULL when no pattern of the batch has an end anchor
  const uint64_t* cand_off; const uint64_t* cand_pre; uint32_t slot0, n_slots;
  const uint32_t* c_doc; const uint64_t* c_off; const uint32_t* c_tf;
  const unsigned long long* list; unsigned long long n;   // list == NULL: candidates 0..n of the group
  uint32_t* scratch;                                      // NULL: shared-memory pass
  unsigned long long* scratch_cursor;
  unsigned long long* ov_list; unsigned long long* ov;    // candidates for the global pass; ov[0] = count, ov[1] = their tf sum
  uint32_t* const* q_bits;                                // per query slot: its docset
  unsigned long long* counters;  // [1] matches [2] format errors [3] positions decoded [4] position bytes
};

__device__ __forceinline__ uint32_t pt_sat_sub(uint32_t a, uint32_t b) { return a > b ? a - b : 0u; }

// intersection_with_slop(left, right, slop) into right[0..): returns the kept length
__device__ uint32_t pt_filter(const uint32_t* left, uint32_t ln, uint32_t* right, uint32_t rn, uint32_t slop, uint32_t lane) {
  uint32_t kept = 0;
  for (uint32_t base = 0; base < rn; base += 32) {
    const uint32_t i = base + lane;
    bool keep = false; uint32_t r = 0;
    if (i < rn) {
      r = right[i];
      uint32_t lo = 0, hi = ln;   // first l > r
      while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (left[mid] <= r) lo = mid + 1; else hi = mid; }
      keep = lo > 0 && left[lo - 1] >= pt_sat_sub(r, slop);
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    __syncwarp();                 // every lane has read its r before the chunk is overwritten
    if (keep) right[kept + __popc(m & ((1u << lane) - 1u))] = r;
    kept += __popc(m);
    __syncwarp();
  }
  return kept;
}

__global__ void __launch_bounds__(PT_WARPS * 32) k_pattern_verify(const PtParams P) {
  __shared__ __align__(16) uint32_t s_buf[PT_WARPS][PT_SMEM_WORDS];
  __shared__ uint32_t s_tail[PT_WARPS][128];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned long long n_match = 0, n_dec = 0, n_bytes = 0;
  bool bad = false;
  for (unsigned long long it = (unsigned long long)blockIdx.x * PT_WARPS + warp; it < P.n; it += (unsigned long long)gridDim.x * PT_WARPS) {
    const unsigned long long c = P.list ? P.list[it] : it;
    uint32_t lo = 0, hi = P.n_slots;   // the slot s with cand_pre[s] <= c < cand_pre[s + 1]
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (P.cand_pre[mid] <= c) lo = mid; else hi = mid; }
    const uint32_t slot = P.slot0 + lo;
    const uint64_t e = P.cand_off[slot] + (c - P.cand_pre[lo]);
    const uint32_t T = P.q_nterms[slot], NP = P.q_nparts[slot];
    uint32_t tf[MAXT], st[MAXT], col[MAXT];
    uint64_t S = 0;
    for (uint32_t t = 0; t < T; t++) { col[t] = P.q_col[(size_t)slot * P.nt + t]; tf[t] = P.c_tf[e * P.nt + col[t]]; st[t] = (uint32_t)S; S += tf[t]; }
    uint32_t* buf;
    if (!P.scratch) {
      if (S > PT_SMEM_WORDS) {
        if (lane == 0) { const unsigned long long i = atomicAdd(P.ov + 0, 1ull); P.ov_list[i] = c; atomicAdd(P.ov + 1, (unsigned long long)S); }
        continue;
      }
      buf = s_buf[warp];
    } else {
      unsigned long long off = 0;
      if (lane == 0) off = atomicAdd(P.scratch_cursor, (unsigned long long)S);
      buf = P.scratch + __shfl_sync(0xffffffffu, off, 0);
    }
    bool ok = true;
    uint64_t cand_bytes = 0;
    for (uint32_t t = 0; t < T; t++) {
      const uint32_t ord = P.q_terms[(size_t)slot * P.nt + col[t]];
      const uint64_t o = P.c_off[e * P.nt + col[t]];
      if (o + tf[t] > P.V.count[ord]) { ok = false; break; }   // the skip entries' tf sums disagree with the positions file
      cand_bytes += ph_read_deltas(P.V, ord, o, tf[t], buf + st[t], s_tail[warp], lane);
      ph_prefix(buf + st[t], tf[t], 0u, lane);
    }
    if (!ok) { bad = true; continue; }
    const uint32_t doc = P.c_doc[e];
    const uint32_t first0 = buf[0], last_raw = buf[st[T - 1] + tf[T - 1] - 1];   // before any filtering
    __syncwarp();   // a pattern without a second term reads buf no more: no lane may overwrite it with the next candidate first
    const uint32_t* left = buf; uint32_t ln = tf[0];
    uint32_t cur = 0, slop = 1;
    bool match = true;
    for (uint32_t i = 0; i < NP && match; i++) {
      const uint32_t part = P.q_parts[(size_t)slot * P.np + i];
      if (part == SB200_PART_TERM) {
        if (cur == 0) { cur = 1; continue; }
        uint32_t* right = buf + st[cur];
        ln = pt_filter(left, ln, right, tf[cur], slop, lane);
        left = right; slop = 1; cur++;
        if (ln == 0) match = false;
      } else if (part == SB200_PART_WILDCARD) {
        slop = 0xFFFFFFFFu;
      } else if (i == 0) {
        if (first0 != 0) match = false;
      } else if (i == NP - 1) {
        if (last_raw != (uint32_t)(P.token_counts[doc] - 1ull)) match = false;
      }
    }
    n_dec += S; n_bytes += cand_bytes;
    if (match) {
      if (lane == 0) atomicOr(P.q_bits[slot] + (doc >> 5), 1u << (doc & 31u));
      n_match++;
    }
  }
  if (lane == 0) {
    if (n_match) atomicAdd(P.counters + 1, n_match);
    if (bad) atomicAdd(P.counters + 2, 1ull);
    if (n_dec) atomicAdd(P.counters + 3, n_dec);
    if (n_bytes) atomicAdd(P.counters + 4, n_bytes);
  }
}

}  // namespace sb200
