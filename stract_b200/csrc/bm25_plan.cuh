// bm25_plan.cuh -- the recall docset of Stract's query plan (core/src/query/plan/, compiled by Query::parse to a tantivy
// BooleanQuery, core/src/query/mod.rs:106-122) and the multi-field recall stage over exactly that docset.
//
// A query's plan is a post-order program of TERM / PHRASE / EMPTY leaves and BOOL nodes (sb200_recall_plan_batch).  Its
// docset follows BooleanWeight (tantivy/src/query/boolean_query/boolean_weight.rs:107-180) with scoring disabled: no clauses
// -> empty; one MustNot clause alone -> empty; one other clause -> that clause; otherwise (Must intersection, or else Should
// union) minus the MustNot union, empty when there is neither Must nor Should.  A phrase leaf matches by
// PhraseScorer::phrase_exists: before the stage, k_phrase_cand<2> + k_phrase_verify in exists mode (bm25_phrase.cuh) build
// the ascending matching documents of every distinct phrase of the batch once.
//
// Docset stage, per group of queries whose candidates fit a memory budget:
//   k_plan_cover   one warp per 128-doc block of a cover posting list writes (query, doc) keys.  The cover of a plan is a
//                  superset of its docset chosen on the host: a TERM's postings, the postings of a PHRASE's rarest term,
//                  the cheapest Must clause of a BOOL (least total doc_freq), or else the union of its Should clauses;
//   radix sort     of the keys (CUB), so each query's candidates ascend and duplicates are adjacent;
//   k_plan_eval    one warp per 32 consecutive candidates of one query runs the whole program on them: a TERM leaf is a
//                  membership probe (block directory search, one block decode, a binary search per lane), a PHRASE leaf a
//                  binary search in that phrase's matching documents, and a BOOL combines its children's ballots;
//   select         (CUB) keeps the first copy of every candidate that the program accepts.
// Recall stage: k_plan_recall, one warp per query, walks its ascending docset 32 documents at a time and seeks every slot's
// cursor forward to them (the posting_contains seek of TextFieldData, core/src/ranking/computer/mod.rs:61-163), then scores
// each document with m_total (bm25_multi.cuh) -- the op program of k_sig_multi -- and keeps the top k by (total desc, doc asc).
#pragma once

namespace sb200 {

constexpr uint32_t PL_MAX_NODES = 256;   // per query; also the deepest evaluation stack
constexpr int PL_WARPS = 4;

struct PSeg { SegView S; const uint4* a128; const uint64_t* t_aoff; uint32_t n_terms, _pad; };
struct PCover { uint32_t q, seg, ord, blk; uint64_t out; };   // one 128-doc block of a cover posting list

__device__ __forceinline__ OTerm pl_term(const PSeg& G, uint32_t ord) {
  OTerm c;
  memset(&c, 0, sizeof(c));
  if (ord < G.n_terms) {
    c.first = G.S.t_first[ord]; c.df = G.S.t_df[ord]; c.nfull = c.df >> 7;
    c.adata = G.t_aoff[ord]; c.end_off = G.S.t_end_off[ord];
    c.tail_off = G.S.t_data_off[ord] + G.S.b_off[c.first + c.nfull];
  }
  return c;
}

// Seeks term c to the documents d of the lanes with `want` (ascending across the lanes) and returns the posting's term
// frequency, 0 when the term does not hold d, or PL_BAD when the directory and the block contents disagree.  *cur / *cached
// (shared memory) are the warp's cursor -- a block index that only moves forward -- and the block held in docs / tfs; they
// persist between calls for the same term.
// POS observes the seek: block(tfs, lane) after every block decode (the whole warp), hit(j, jj) when a lane finds d at entry jj
// of block j.  pl_seek itself observes nothing; k_wp_signals (bm25_webpage.cuh) records position offsets this way.
constexpr uint64_t PL_BAD = 1ull << 32;
struct PlNoPos {
  __device__ __forceinline__ void block(const uint32_t*, uint32_t) {}
  __device__ __forceinline__ void hit(uint32_t, uint32_t) {}
};
template <class POS>
__device__ __forceinline__ uint64_t pl_seek_at(const PSeg& G, const OTerm& c, uint32_t* cur_p, uint32_t* cached_p, uint32_t* docs, uint32_t* tfs,
                                               uint32_t* bloom, uint32_t d, bool want, uint32_t lane, POS& pos) {
  uint32_t cur = *cur_p, cached = *cached_p, tf = 0;
  bool pend = want && c.df > 0, bad = false;
  for (uint32_t guard = 0;; guard++) {
    const uint32_t m = __reduce_min_sync(0xffffffffu, pend ? d : 0xFFFFFFFFu);
    if (m == 0xFFFFFFFFu) break;
    if (guard > 64u) { bad = true; break; }
    const uint32_t j = o3_dir_search(G.S.b_last + c.first, cur, c.nfull, m, lane);
    if (j == c.nfull && (c.df & 127u) == 0) break;     // past the last block: nothing left to find
    cur = j;
    if (j != cached) {
      uint32_t last;
      const uint32_t prev = j ? __ldg(G.S.b_last + c.first + j - 1) : 0u;
      o3_decode(G.S, G.a128, c, j, prev, docs, tfs, bloom, lane, last);
      cached = j;
      __syncwarp();
      pos.block(tfs, lane);
    }
    const uint32_t lastB = j < c.nfull ? docs[127] : 0xFFFFFFFFu;   // the tail decides everything that is left
    if (pend && d <= lastB) {
      pend = false;
      const uint32_t jj = lower_bound128(docs, d);
      if (jj < 128u && docs[jj] == d) { tf = tfs[jj]; pos.hit(j, jj); }
    }
  }
  __syncwarp();
  if (lane == 0) { *cur_p = cur; *cached_p = cached; }
  __syncwarp();
  return bad ? PL_BAD : (uint64_t)tf;
}
__device__ uint64_t pl_seek(const PSeg& G, const OTerm& c, uint32_t* cur_p, uint32_t* cached_p, uint32_t* docs, uint32_t* tfs, uint32_t* bloom,
                            uint32_t d, bool want, uint32_t lane) {
  PlNoPos none;
  return pl_seek_at(G, c, cur_p, cached_p, docs, tfs, bloom, d, want, lane, none);
}

struct PlanParams {
  const PSeg* segs;
  const sb200_plan_node* nodes; const uint32_t* node_off;   // per query of the group: its program
  const PCover* cover; uint32_t n_cover;
  const uint32_t* ph_off; const uint32_t* ph_docs;          // per distinct phrase: its ascending matching documents
  const uint64_t* keys; uint64_t n_keys;                    // sorted (query << 32 | doc)
  const uint64_t* q_beg;                                    // [n_q + 1] the group's queries' ranges in keys
  const uint32_t* units; uint32_t n_units;                  // k_plan_eval: first key of every 32-key chunk
  uint8_t* keep;
  unsigned long long* counters;                              // [2] format errors
};

// one warp per cover block: decode it, write the (query, doc) keys
__global__ void __launch_bounds__(PL_WARPS * 32) k_plan_cover(const PlanParams P) {
  __shared__ __align__(16) uint32_t s_docs[PL_WARPS][128], s_tfs[PL_WARPS][128], s_bloom[PL_WARPS][16];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t u = blockIdx.x * PL_WARPS + warp;
  if (u >= P.n_cover) return;
  const PCover C = P.cover[u];
  const PSeg& G = P.segs[C.seg];
  const OTerm c = pl_term(G, C.ord);
  const uint32_t prev = C.blk ? __ldg(G.S.b_last + c.first + C.blk - 1) : 0u;
  uint32_t last;
  const uint32_t n = o3_decode(G.S, G.a128, c, C.blk, prev, s_docs[warp], s_tfs[warp], s_bloom[warp], lane, last);
  __syncwarp();
  bool bad = false;
  for (uint32_t i = lane; i < n; i += 32) {
    const uint32_t d = s_docs[warp][i];
    if (d >= G.S.max_doc) bad = true;
    ((unsigned long long*)P.keys)[C.out + i] = ((unsigned long long)C.q << 32) | (bad ? 0u : d);
  }
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicAdd(P.counters + 2, 1ull);
}

// one warp per chunk of <= 32 sorted keys of one query: keep[i] = first copy of the doc and the program accepts it
__global__ void __launch_bounds__(PL_WARPS * 32) k_plan_eval(const PlanParams P) {
  __shared__ __align__(16) uint32_t s_docs[PL_WARPS][128], s_tfs[PL_WARPS][128], s_bloom[PL_WARPS][16];
  __shared__ uint32_t s_mask[PL_WARPS][PL_MAX_NODES];
  __shared__ uint8_t s_occ[PL_WARPS][PL_MAX_NODES];
  __shared__ uint32_t s_cur[PL_WARPS][2];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t u = blockIdx.x * PL_WARPS + warp;
  if (u >= P.n_units) return;
  const uint64_t first = P.units[u];       // a chunk never crosses a query
  const uint64_t key0 = P.keys[first];
  const uint32_t q = (uint32_t)(key0 >> 32);
  const uint64_t qend = P.q_beg[q + 1];
  const uint64_t at = first + lane;
  const bool live = at < qend && at < first + 32;
  const uint32_t d = live ? (uint32_t)P.keys[at] : 0xFFFFFFFFu;
  const bool dup = live && at > P.q_beg[q] && (uint32_t)P.keys[at - 1] == d;
  uint32_t* mask = s_mask[warp]; uint8_t* occ = s_occ[warp];
  uint32_t sp = 0;
  bool bad = false;
  const uint32_t n0 = P.node_off[q], n1 = P.node_off[q + 1];
  for (uint32_t x = n0; x < n1; x++) {
    const sb200_plan_node N = P.nodes[x];
    uint32_t m = 0;
    if (N.kind == SB200_PLAN_TERM) {
      if (N.arg != SB200_ABSENT_TERM) {
        const PSeg& G = P.segs[N.segment];
        const OTerm c = pl_term(G, N.arg);
        if (lane == 0) { s_cur[warp][0] = 0; s_cur[warp][1] = 0xFFFFFFFFu; }
        __syncwarp();
        const uint64_t r = pl_seek(G, c, &s_cur[warp][0], &s_cur[warp][1], s_docs[warp], s_tfs[warp], s_bloom[warp], d, live && !dup, lane);
        if (r == PL_BAD) bad = true;
        m = __ballot_sync(0xffffffffu, r != 0 && r != PL_BAD);
      }

    } else if (N.kind == SB200_PLAN_PHRASE) {   // arg: the distinct phrase; a binary search in its matching documents
      bool hit = false;
      if (live && !dup) {
        uint32_t lo = P.ph_off[N.arg], hi = P.ph_off[N.arg + 1];
        const uint32_t end = hi;
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (P.ph_docs[mid] < d) lo = mid + 1; else hi = mid; }
        hit = lo < end && P.ph_docs[lo] == d;
      }
      m = __ballot_sync(0xffffffffu, hit);
    } else if (N.kind == SB200_PLAN_BOOL) {
      const uint32_t nc = N.n_children, b = sp - nc;
      uint32_t must = 0xFFFFFFFFu, should = 0, nots = 0;
      bool has_must = false, has_should = false;
      for (uint32_t c = b; c < sp; c++) {
        if (occ[c] == SB200_PLAN_MUST) { must &= mask[c]; has_must = true; }
        else if (occ[c] == SB200_PLAN_SHOULD) { should |= mask[c]; has_should = true; }
        else nots |= mask[c];
      }
      if (nc == 1) m = occ[b] == SB200_PLAN_MUST_NOT ? 0u : mask[b];
      else if (nc > 1) m = (has_must ? must : (has_should ? should : 0u)) & ~nots;
      sp = b;
    }
    __syncwarp();
    if (lane == 0) { mask[sp] = m; occ[sp] = N.occur; }
    sp++;
    __syncwarp();
  }
  const bool ok = live && !dup && ((mask[0] >> lane) & 1u);
  if (live) P.keep[at] = ok ? 1 : 0;
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicAdd(P.counters + 2, 1ull);
}

// q_beg[q] = first key of query q (lower bound of q << 32), q_beg[n] = n_keys
__global__ void k_plan_bounds(const uint64_t* __restrict__ keys, uint64_t n_keys, uint32_t n, uint64_t* q_beg) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q > n) return;
  const uint64_t x = (uint64_t)q << 32;
  uint64_t lo = 0, hi = n_keys;
  while (lo < hi) { const uint64_t mid = (lo + hi) >> 1; if (keys[mid] < x) lo = mid + 1; else hi = mid; }
  q_beg[q] = q == n ? n_keys : lo;
}

// the low 32 bits of keys[0, n) (the docs of a group's docset, query by query)
__global__ void k_plan_docs(const uint64_t* __restrict__ keys, uint64_t n, uint32_t* out) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = (uint32_t)keys[i];
}

// ------------------------------------------------------------------ recall stage --------------------------------------------
template <int TMAX>
__host__ __device__ constexpr size_t pl_warp_smem() { return (size_t)TMAX * 128 * 8 + (size_t)TMAX * 16 * 4 + (size_t)TMAX * sizeof(OTerm) + (size_t)TMAX * 16 + 16 * 4; }
template <int TMAX>
__host__ __device__ constexpr size_t pl_cta_smem() { return M_MAX_FIELDS * 256 * 4 + M_MAX_OPS * sizeof(MOp) + WQ * pl_warp_smem<TMAX>(); }

struct PlanRecallParams {
  MParams M;                     // fields, ops, slots (per group query, text slots first), optic tables by M.q_orig
  const uint64_t* keys; const uint64_t* q_beg;   // the group's docsets
};

// one warp per query: walk its ascending docset 32 documents at a time (lane i holds the i-th); the whole warp seeks every slot
// to the 32 documents (pl_seek), then every lane scores its own
template <int TMAX>
__global__ void __launch_bounds__(WQ * 32) k_plan_recall(const PlanRecallParams R) {
  const MParams& P = R.M;
  SB_DYN_SMEM(smem_raw);
  float* s_cache = (float*)smem_raw;                                   // [M_MAX_FIELDS][256]
  MOp* s_ops = (MOp*)(smem_raw + M_MAX_FIELDS * 256 * 4);              // [M_MAX_OPS]
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char* wbase = smem_raw + M_MAX_FIELDS * 256 * 4 + M_MAX_OPS * sizeof(MOp) + warp * pl_warp_smem<TMAX>();
  uint32_t* docs = (uint32_t*)wbase;                                   // [TMAX][128]
  uint32_t* tfs = docs + TMAX * 128;                                   // [TMAX][128]
  uint32_t* bloom = tfs + TMAX * 128;                                  // [TMAX][16]
  OTerm* tc = (OTerm*)(bloom + TMAX * 16);                             // [TMAX]
  float* s_wf = (float*)(tc + TMAX);                                   // [TMAX]
  uint32_t* s_fld = (uint32_t*)(s_wf + TMAX);                          // [TMAX]
  uint32_t* s_cur = s_fld + TMAX;                                      // [TMAX]
  uint32_t* s_cached = s_cur + TMAX;                                   // [TMAX]
  uint32_t* s_nf = s_cached + TMAX;                                    // [M_MAX_FIELDS]
  uint32_t* s_count = s_nf + 8;
  for (uint32_t i = threadIdx.x; i < P.n_fields * 256; i += WQ * 32) s_cache[i] = P.fields[i >> 8].cache[i & 255];
  for (uint32_t i = threadIdx.x; i < P.n_ops; i += WQ * 32) s_ops[i] = P.ops[i];
  __syncthreads();  // the only block barrier
  const uint32_t q = blockIdx.x * WQ + warp;
  if (q >= P.n_queries) return;
  const uint32_t SM = P.n_slots_max;
  const uint32_t oq = P.q_orig[q];
  const uint32_t T = min(P.q_nslots[q], (uint32_t)TMAX);
  uint64_t* khi = P.g_khi + (size_t)q * P.cap; uint32_t* klo = P.g_klo + (size_t)q * P.cap;
  const uint32_t* o_ex = nullptr; const uint32_t* o_rq = nullptr;
  const uint32_t ex = P.d_exclude ? P.d_exclude[oq] : SB200_NO_DOCSET, rq = P.d_require ? P.d_require[oq] : SB200_NO_DOCSET;
  if (ex != SB200_NO_DOCSET) o_ex = P.d_bits[ex];
  if (rq != SB200_NO_DOCSET) o_rq = P.d_bits[rq];
  const uint32_t o_nr = P.d_nrules ? P.d_nrules[oq] : 0u;
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
  if (lane == 0) *s_count = 0;
  __syncwarp();
  bool thr_on = false; uint64_t thr_hi = 0; uint32_t thr_lo = 0;   // warp-uniform
  unsigned long long my_docs = 0;
  bool bad = false;
  const uint64_t beg = R.q_beg[q], end = R.q_beg[q + 1];
  for (uint64_t base = beg; base < end; base += 32) {
    const bool live = base + lane < end;
    const uint32_t d = live ? (uint32_t)R.keys[base + lane] : 0xFFFFFFFFu;
    bool take = live && d < P.max_doc;
    if (live && !take) bad = true;
    if (take && o_ex && m_in(o_ex, d)) take = false;   // Discard rules, blocked hosts
    if (take && o_rq && !m_in(o_rq, d)) take = false;  // DiscardNonMatching
    uint32_t tf[TMAX];
#pragma unroll
    for (int x = 0; x < TMAX; x++) {
      tf[x] = 0;
      if ((uint32_t)x >= T) continue;
      const MField& F = P.fields[s_fld[x] & 0x7Fu];
      PSeg G; G.S = F.S; G.a128 = F.a128; G.t_aoff = F.t_aoff; G.n_terms = F.n_terms;
      const uint64_t r = pl_seek(G, tc[x], s_cur + x, s_cached + x, docs + x * 128, tfs + x * 128, bloom + x * 16, d, take, lane);
      if (r == PL_BAD) bad = true; else tf[x] = (uint32_t)r;
    }
    // room for 32 more entries: keep the best k so far and raise the threshold
    const uint32_t have = *s_count;
    __syncwarp();
    if (have + 32 > P.cap) {
      w_sort_prefix_desc(khi, klo, have, P.cap, lane);
      const uint32_t c = min(have, P.k);
      if (c == P.k) { thr_on = true; thr_hi = khi[P.k - 1]; thr_lo = klo[P.k - 1]; }
      __syncwarp();
      if (lane == 0) *s_count = c;
      __syncwarp();
    }
    if (take) {
      my_docs++;
      MNoSink none;
      const double total = m_total<TMAX, true>(P, s_ops, s_cache, s_nf, s_fld, s_wf, tc, T, q, d, tf, oq, o_nr, none);
      const uint64_t kh = ord_f64(total);
      const uint32_t kl = ~d;
      if (!thr_on || key_gt(kh, kl, thr_hi, thr_lo)) {
        const uint32_t at = atomicAdd(s_count, 1u);
        khi[at] = kh; klo[at] = kl;
      }
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
  const bool any_bad = __any_sync(0xffffffffu, bad);
  if (lane == 0) {
    if (my_docs) atomicAdd(P.counters + 0, my_docs);
    if (any_bad) atomicAdd(P.counters + 2, 1ull);
  }
}

}  // namespace sb200
