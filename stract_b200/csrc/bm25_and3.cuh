// bm25_and3.cuh -- AND queries, third generation (bit-identical to k_topk_warp<AND>, which keeps only the batches
// with a single-clause query above 65 536 postings).
//
// Why: a CPU emulation of k_topk_warp<AND> on the C4 batch (10k 2-term queries) counts 4.1 M rounds of ~250 per
// work item, evenly spread -- no tail -- and a round there is ~1500
// serial instructions of generic T-term bookkeeping on cursor structs in shared memory; the memory system is idle.
// The intersection itself needs far less:
//   * work unit = (query, a few consecutive 128-doc blocks of its RAREST term A); one warp per unit.  Units are
//     independent, uniform and plentiful (~150 k on C4), so no LPT ordering, doc-range split or merge pass;
//   * the A block stays in registers (4 docs per lane).  For every other term X (in doc_freq order, like
//     tantivy's Intersection) the warp looks up, through the block directory, the one X block that can hold the
//     smallest undecided A doc (32-wide hop, then 32-ary search: <= 3 dependent loads instead of a linear walk),
//     decodes ONLY its doc ids into shared memory, and every lane binary-searches its undecided docs in it;
//   * term frequencies are not unpacked at all: a hit reads its tf straight out of the packed stream (hits are
//     ~1 % of the probes), the fieldnorm byte is fetched for hits only;
//   * an AND result is a subset of A, so a query's candidate list has a hard capacity of doc_freq(A): hits are
//     appended with one warp-aggregated atomic per A block, no threshold, no overflow path.  k_and3_select then
//     takes the exact top-k per query (score desc, doc asc) in shared memory, chunk-wise for long lists.
// Scores follow Intersection::score (intersection.rs:153-157): (left + right) + sum(others), f32, same rounding
// intrinsics as k_topk_warp, so results are bit-identical to it.
#pragma once

namespace sb200 {

constexpr int A3_WARPS = 4;              // units (warps) per CTA
constexpr uint32_t A3_UNIT_BLOCKS = 4;   // A blocks per unit
constexpr uint32_t A3_SEL_CAP = 8192;    // select kernel: entries in shared memory (>= 2 * SB200_MAX_K)
static_assert(A3_SEL_CAP >= 2 * SB200_MAX_K, "select buffer must hold the kept k plus at least k new entries");

struct AUnit { uint32_t q, blk_lo, blk_hi, _pad; };

struct A3Params {
  SegView S;
  const uint4* a128; const uint64_t* t_aoff;
  const uint32_t* q_terms; const uint32_t* q_nterms; const float* q_weights; const float* cache;
  uint32_t n_terms_max;
  const AUnit* units; uint32_t n_units;
  const uint64_t* cand_off;   // per query slot: start of its candidate list
  uint32_t* cand_cnt;         // per query slot: entries appended so far
  uint32_t* c_key; uint32_t* c_doc;
  unsigned long long* counters;
};

struct A3Term { uint32_t first, nfull, df; uint64_t adata, tail_off, end_off; float weight; };  // warp-uniform
struct A3Blk { const uint4* base; uint32_t db, tb, strict; };                                   // a packed block

__device__ __forceinline__ A3Term a3_load_term(const A3Params& P, uint32_t q, uint32_t slot) {
  const SegView& S = P.S;
  A3Term t;
  const uint32_t ord = P.q_terms[(size_t)q * P.n_terms_max + slot];
  t.first = S.t_first[ord]; t.df = S.t_df[ord]; t.nfull = t.df >> 7;
  t.adata = P.t_aoff[ord]; t.end_off = S.t_end_off[ord];
  t.tail_off = S.t_data_off[ord] + S.b_off[t.first + t.nfull];
  t.weight = P.q_weights[(size_t)q * P.n_terms_max + slot];
  return t;
}

// docs 4*lane .. 4*lane+3 of full block `blk`; B describes the packed block for later tf reads
__device__ __forceinline__ uint4 a3_decode_docs(const A3Params& P, const A3Term& t, uint32_t blk, uint32_t lane, A3Blk& B) {
  const SegView& S = P.S;
  const uint32_t idx = t.first + blk;
  const uint32_t bits = S.b_bits[idx];
  B.db = bits & 0x3fu; B.strict = (bits >> 6) & 1u; B.tb = bits >> 8;
  B.base = P.a128 + t.adata + (S.b_off[idx] >> 4);
  const uint32_t prev_last = blk ? S.b_last[idx - 1] : 0u;
  uint4 d = unpack4(B.base, B.db, lane);
  const uint32_t st = B.strict;
  d.x += st; d.y += d.x + st; d.z += d.y + st; d.w += d.z + st;   // lane-local inclusive sums of the deltas
  const uint32_t incl = warp_scan_incl(d.w, lane);
  const uint32_t before = incl - d.w + ((st && prev_last == 0) ? 0xFFFFFFFFu : prev_last);  // offset 0 == None
  d.x += before; d.y += before; d.z += before; d.w += before;
  return d;
}

// term frequency of posting k (0..127) of a packed block, read straight from the bit stream
__device__ __forceinline__ uint32_t a3_tf_at(const SegView& S, const A3Blk& B, uint32_t k) {
  if (S.record < 1) return 1u;
  if (B.tb == 0) return B.strict;
  const uint32_t* words = (const uint32_t*)(B.base + B.db);
  const uint32_t l4 = k & 3u, bit = (k >> 2) * B.tb, w = bit >> 5, sh = bit & 31u;
  const uint32_t lo = __ldg(words + w * 4 + l4);
  const uint32_t hi = (sh + B.tb > 32) ? __ldg(words + (w + 1) * 4 + l4) : 0u;
  const uint32_t v = __funnelshift_r(lo, hi, sh);
  return ((B.tb == 32) ? v : (v & ((1u << B.tb) - 1u))) + B.strict;
}

// vint tail of term t (compression/vint.rs) into sd/stf[128]; entries >= n hold TERMINATED / 1; returns n
__device__ uint32_t a3_decode_tail(const A3Params& P, const A3Term& t, uint32_t* sd, uint32_t* stf, uint32_t lane) {
  const SegView& S = P.S;
  const uint32_t n = t.df - t.nfull * 128u;
  const uint32_t prev_last = t.nfull ? S.b_last[t.first + t.nfull - 1] : 0u;
  const uint8_t* bytes = (const uint8_t*)S.p32 + t.tail_off;
  const uint32_t nbytes = (uint32_t)min((uint64_t)1340, t.end_off - t.tail_off);
  __syncwarp();
  for (uint32_t i = lane; i < 128; i += 32) { sd[i] = 0; stf[i] = 1; }
  __syncwarp();
  uint32_t seen = 0;
  const uint32_t want = (S.record >= 1) ? 2 * n : n;
  for (uint32_t base = 0; base < nbytes && seen < want; base += 32) {
    const uint32_t b = base + lane;
    const uint32_t byte = (b < nbytes) ? bytes[b] : 0u;
    const bool stop = (byte & 0x80u) != 0;
    const unsigned m = __ballot_sync(0xffffffffu, stop);
    if (stop) {
      const uint32_t idx = seen + __popc(m & ((1u << lane) - 1u));
      if (idx < want) {
        uint32_t v = byte & 0x7Fu, start = b;
        while (start > 0 && b - start < 4 && !(bytes[start - 1] & 0x80u)) { start--; v = (v << 7) | (bytes[start] & 0x7Fu); }
        if (idx < n) sd[idx] = v; else stf[idx - n] = v;
      }
    }
    seen += __popc(m);
  }
  __syncwarp();
  uint4 d = ((uint4*)sd)[lane];
  d.y += d.x; d.z += d.y; d.w += d.z;
  const uint32_t incl = warp_scan_incl(d.w, lane);
  const uint32_t before = incl - d.w + prev_last;
  d.x += before; d.y += before; d.z += before; d.w += before;
  const uint32_t k0 = lane * 4;
  if (k0 + 0 >= n) d.x = TERMINATED;
  if (k0 + 1 >= n) d.y = TERMINATED;
  if (k0 + 2 >= n) d.z = TERMINATED;
  if (k0 + 3 >= n) d.w = TERMINATED;
  __syncwarp();
  ((uint4*)sd)[lane] = d;
  __syncwarp();
  return n;
}

// smallest full-block index j in [from, nfull) whose last doc is >= dmin, nfull if there is none.  A 32-wide hop
// over the next entries first (the common case while a unit walks forward), then a 32-ary search.
__device__ __forceinline__ uint32_t a3_dir_search(const SegView& S, const A3Term& t, uint32_t from, uint32_t dmin, uint32_t lane) {
  const uint32_t* __restrict__ last = S.b_last + t.first;
  uint32_t lo = from, hi = t.nfull;
  if (lo >= hi) return hi;
  {
    const uint32_t idx = lo + lane;
    const bool pred = idx >= hi || __ldg(last + idx) >= dmin;
    const unsigned m = __ballot_sync(0xffffffffu, pred);
    if (m) return min(lo + (uint32_t)__ffs(m) - 1u, hi);
    lo += 32;
  }
  while (lo < hi) {  // invariant: every j < lo has last[j] < dmin; the answer is in [lo, hi]
    const uint32_t span = hi - lo, step = (span + 31u) / 32u;
    const uint32_t cs = lo + lane * step;                       // this lane's chunk [cs, cs + step)
    const bool empty = cs >= hi;
    const uint32_t e = empty ? 0u : min(cs + step - 1u, hi - 1u);
    const bool pred = empty || __ldg(last + e) >= dmin;
    const unsigned m = __ballot_sync(0xffffffffu, pred);
    if (!m) return hi;
    const uint32_t fcs = lo + ((uint32_t)__ffs(m) - 1u) * step;
    if (fcs >= hi) return hi;                                   // the first "true" chunk is an empty one
    lo = fcs; hi = min(fcs + step - 1u, hi - 1u);               // last[hi] >= dmin: answer in [lo, hi]
  }
  return lo;
}

__device__ __forceinline__ float a3_term_score(float weight, uint32_t tf, float norm) {
  const float t = (float)tf;
  return __fmul_rn(weight, __fdiv_rn(t, __fadd_rn(t, norm)));   // Bm25Weight::score, bm25.rs:182-196
}

// At least 8 resident CTAs per SM caps the registers at 64, with a small spill (5 CTAs would allow 96 and no spill,
// 6 would allow 80).  The kernel lives on latency hiding, so occupancy wins.
__global__ void __launch_bounds__(A3_WARPS * 32, 8) k_and3(const A3Params P) {
  __shared__ float cache[256];
  __shared__ __align__(16) uint32_t s_docs[A3_WARPS][128];
  __shared__ __align__(16) uint32_t s_tfs[A3_WARPS][128];
  __shared__ uint32_t s_cur[A3_WARPS][MAXT];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (uint32_t i = threadIdx.x; i < 256; i += A3_WARPS * 32) cache[i] = P.cache[i];
  __syncthreads();  // the only block barrier
  const uint32_t u = blockIdx.x * A3_WARPS + warp;
  if (u >= P.n_units) return;
  const SegView& S = P.S;
  const AUnit U = P.units[u];
  const uint32_t q = U.q, T = P.q_nterms[q];
  uint32_t* sd = s_docs[warp]; uint32_t* stf = s_tfs[warp]; uint32_t* cur = s_cur[warp];
  if (lane < MAXT) cur[lane] = 0;
  __syncwarp();
  if (T == 0) return;
  const A3Term tA = a3_load_term(P, q, 0);
  unsigned long long n_blocks = 0, n_hits = 0;
  bool watchdog = false, bad_doc = false;

  for (uint32_t ablk = U.blk_lo; ablk < U.blk_hi; ablk++) {
    // ---- this lane's four docs of the A block
    uint32_t d[4], tfa[4] = {1u, 1u, 1u, 1u};
    A3Blk BA; BA.base = nullptr; BA.db = 0; BA.tb = 0; BA.strict = 0;
    bool a_tail = false; uint32_t nA = 128;
    if (ablk < tA.nfull) {
      const uint4 v = a3_decode_docs(P, tA, ablk, lane, BA);
      d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
    } else {
      a_tail = true;
      nA = a3_decode_tail(P, tA, sd, stf, lane);
      const uint4 v = ((const uint4*)sd)[lane], f = ((const uint4*)stf)[lane];
      d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
      tfa[0] = f.x; tfa[1] = f.y; tfa[2] = f.z; tfa[3] = f.w;
      __syncwarp();
    }
    n_blocks++;
    uint32_t alive = 0;
#pragma unroll
    for (int b = 0; b < 4; b++) if (lane * 4 + b < nA) {
      if (d[b] < S.max_doc) alive |= 1u << b;
      else bad_doc = true;   // corrupt deltas: never index the doc tables with it
    }
    float nrm[4] = {0.f, 0.f, 0.f, 0.f}, acc[4] = {0.f, 0.f, 0.f, 0.f}, oth[4] = {0.f, 0.f, 0.f, 0.f};

    // ---- every other clause, rarest first; only the survivors of clause x-1 are looked up in clause x
    for (uint32_t x = 1; x < T; x++) {
      if (!__any_sync(0xffffffffu, alive != 0)) break;
      const A3Term tX = a3_load_term(P, q, x);
      uint32_t pend = alive;
      uint32_t tfx[4] = {0u, 0u, 0u, 0u};
      // every pass decides at least the smallest undecided doc (<= 128 of them); more passes mean the directory
      // and the block contents disagree -- fail the batch instead of spinning
      for (uint32_t guard = 0;; guard++) {
        if (guard > 130u) { watchdog = true; break; }
        uint32_t m = 0xFFFFFFFFu;   // smallest undecided doc of the warp (a lane's docs ascend with b)
#pragma unroll
        for (int b = 3; b >= 0; b--) if ((pend >> b) & 1u) m = d[b];
#pragma unroll
        for (int o = 16; o; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (m == 0xFFFFFFFFu) break;
        const uint32_t from = cur[x];
        const uint32_t jb = a3_dir_search(S, tX, from, m, lane);
        __syncwarp();
        if (lane == 0) cur[x] = jb;
        uint32_t lastB, lenB; bool x_tail = false;
        A3Blk BX; BX.base = nullptr; BX.db = 0; BX.tb = 0; BX.strict = 0;
        if (jb < tX.nfull) {
          const uint4 v = a3_decode_docs(P, tX, jb, lane, BX);
          __syncwarp();                       // every lane is done with the previous contents of sd
          ((uint4*)sd)[lane] = v;
          lastB = __shfl_sync(0xffffffffu, v.w, 31); lenB = 128;
          __syncwarp();
        } else {                              // past the full blocks: the vint tail decides everything that is left
          x_tail = true; lastB = 0xFFFFFFFFu;
          lenB = (tX.df & 127u) ? a3_decode_tail(P, tX, sd, stf, lane) : 0u;
        }
        n_blocks++;
#pragma unroll
        for (int b = 0; b < 4; b++) {
          if (((pend >> b) & 1u) && d[b] <= lastB) {
            pend &= ~(1u << b);
            bool found = false; uint32_t j = 0;
            if (lenB) { j = lower_bound128(sd, d[b]); found = j < lenB && sd[j] == d[b]; }
            if (!found) alive &= ~(1u << b);
            else tfx[b] = x_tail ? stf[j] : a3_tf_at(S, BX, j);
          }
        }
        if (x_tail) break;
      }
      // scores of the survivors (Intersection::score: left + right, then the others in clause order)
#pragma unroll
      for (int b = 0; b < 4; b++) {
        if (!((alive >> b) & 1u)) continue;
        if (x == 1) {
          nrm[b] = cache[S.fieldnorm[d[b]]];
          const uint32_t tf0 = a_tail ? tfa[b] : a3_tf_at(S, BA, lane * 4 + b);
          acc[b] = __fadd_rn(a3_term_score(tA.weight, tf0, nrm[b]), a3_term_score(tX.weight, tfx[b], nrm[b]));
        } else {
          oth[b] = __fadd_rn(oth[b], a3_term_score(tX.weight, tfx[b], nrm[b]));
        }
      }
    }
    if (T == 1) {   // a single clause: every posting is a hit, score = its term score
#pragma unroll
      for (int b = 0; b < 4; b++) if ((alive >> b) & 1u) {
        nrm[b] = cache[S.fieldnorm[d[b]]];
        const uint32_t tf0 = a_tail ? tfa[b] : a3_tf_at(S, BA, lane * 4 + b);
        acc[b] = a3_term_score(tA.weight, tf0, nrm[b]);
      }
    }
    // ---- append the hits to the query's candidate list
    const uint32_t cnt = __popc(alive);
    const uint32_t incl = warp_scan_incl(cnt, lane);
    const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
    if (total) {
      uint32_t base = 0;
      if (lane == 0) base = atomicAdd(P.cand_cnt + q, total);
      base = __shfl_sync(0xffffffffu, base, 0);
      uint64_t pos = P.cand_off[q] + base + (incl - cnt);
#pragma unroll
      for (int b = 0; b < 4; b++) if ((alive >> b) & 1u) {
        const float score = (T == 1) ? acc[b] : __fadd_rn(acc[b], oth[b]);
        P.c_key[pos] = ord_f32(score); P.c_doc[pos] = d[b]; pos++;
      }
      n_hits += total;
    }
    __syncwarp();
  }
  if (__any_sync(0xffffffffu, bad_doc)) watchdog = true;
  if (lane == 0) {
    if (n_hits) atomicAdd(P.counters + 0, n_hits);
    if (n_blocks) atomicAdd(P.counters + 1, n_blocks);
    if (watchdog) atomicAdd(P.counters + 2, 1ull);
  }
}

// exact top-k of every query's candidate list: one CTA per query slot, keys (score bits, ~doc), descending
__global__ void __launch_bounds__(256) k_and3_select(const uint64_t* __restrict__ cand_off, const uint32_t* __restrict__ cand_cnt,
                                                     const uint32_t* __restrict__ c_key, const uint32_t* __restrict__ c_doc,
                                                     const uint32_t* __restrict__ q_orig, uint32_t slot0, uint32_t k,
                                                     uint32_t* o_docs, float* o_scores, uint32_t* o_n) {
  SB_DYN_SMEM(smem_raw);
  uint32_t* kh = (uint32_t*)smem_raw;          // [A3_SEL_CAP]
  uint32_t* kl = kh + A3_SEL_CAP;              // [A3_SEL_CAP]  ~doc
  const uint32_t slot = slot0 + blockIdx.x, tid = threadIdx.x;
  const uint32_t n = cand_cnt[slot];
  const uint64_t off = cand_off[slot];
  uint32_t kept = 0, pos = 0;
  while (pos < n) {
    const uint32_t take = min(n - pos, A3_SEL_CAP - kept);
    for (uint32_t i = tid; i < take; i += 256) { kh[kept + i] = c_key[off + pos + i]; kl[kept + i] = ~c_doc[off + pos + i]; }
    const uint32_t m = kept + take;
    uint32_t n2 = 2; while (n2 < m) n2 <<= 1;
    for (uint32_t i = m + tid; i < n2; i += 256) { kh[i] = 0; kl[i] = 0; }
    for (uint32_t size = 2; size <= n2; size <<= 1) {
      for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
        __syncthreads();
        for (uint32_t i = tid; i < (n2 >> 1); i += 256) {
          const uint32_t lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
          const bool desc = ((lo & size) == 0);
          const uint32_t ah = kh[lo], bh = kh[hi], al = kl[lo], bl = kl[hi];
          const bool a_gt_b = ah > bh || (ah == bh && al > bl);
          const bool b_gt_a = bh > ah || (ah == bh && bl > al);
          if (desc ? b_gt_a : a_gt_b) { kh[lo] = bh; kl[lo] = bl; kh[hi] = ah; kl[hi] = al; }
        }
      }
    }
    __syncthreads();
    kept = min(m, k);
    pos += take;
  }
  const uint32_t oq = q_orig ? q_orig[slot] : slot;
  for (uint32_t i = tid; i < kept; i += 256) {
    o_docs[(size_t)oq * k + i] = ~kl[i];
    o_scores[(size_t)oq * k + i] = unord_f32(kh[i]);
  }
  if (tid == 0) o_n[oq] = kept;
}

}  // namespace sb200
