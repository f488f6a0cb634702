// bm25_or3.cuh -- OR / signal-combine queries, third generation (the union kernel since round 2: bit-identical
// to k_topk_warp<OR|SIGNAL> on hardware, 1.2-1.4x faster).
//
// Same algorithm, work items, candidate buffers, merge pass and bit-exact scoring as k_topk_warp (block-synchronous
// union: bound = smallest last-doc of the current blocks, lowest slot owns a doc, TopNComputer-style threshold),
// rebuilt around what the round-1 numbers say about that kernel: ~750 warp instructions per pass of 32 candidates,
// about half of them round bookkeeping on cursor structs in shared memory, most of the rest failed membership
// searches.  Changes:
//   * the cursor of term t lives in the registers of LANE t (pos, len, last doc, next block, flags).  bound is one
//     redux.sync, the per-term ranges are one parallel lower_bound + one warp scan, refills are driven by a ballot:
//     no per-term loops over shared structs, no lane-0 sections, a third of the __syncwarp()s;
//   * every decoded block gets a 512-bit presence filter (bit = doc mod 512, built with 4 shared atomics per lane).
//     A candidate consults the filter of every other term first and runs the 8-step search only on a hit: with 128
//     docs per block ~78 % of the searches (nearly all of them fail on sparse lists) are skipped;
//   * the kernel is instantiated per term-count bound (2, 3, 5, 8), so the per-candidate loops over terms are
//     unrolled to the batch's width instead of always 8;
//   * doc-range items start through the 32-ary directory search instead of a linear block walk.
// Not covered (falls back to k_topk_warp): the max_docs short-circuit of path B.
#pragma once

namespace sb200 {

constexpr uint32_t O3_STAGE_BYTES = 256;   // a staged block: (doc bits + tf bits) * 16 B <= 256, i.e. <= 16 bits per posting
constexpr uint32_t O3_NONE = 0xFFFFFFFFu;
struct OTerm { uint64_t adata, tail_off, end_off; uint32_t first, nfull, df; float weight; };  // per (warp, term), shared
static_assert(sizeof(OTerm) == 40, "OTerm layout");

// smallest j in [from, nfull) with last[j] >= dmin, nfull if none (same search as a3_dir_search)
__device__ __forceinline__ uint32_t o3_dir_search(const uint32_t* __restrict__ last, uint32_t from, uint32_t nfull, uint32_t dmin, uint32_t lane) {
  uint32_t lo = from, hi = nfull;
  if (lo >= hi) return hi;
  {
    const uint32_t idx = lo + lane;
    const bool pred = idx >= hi || __ldg(last + idx) >= dmin;
    const unsigned m = __ballot_sync(0xffffffffu, pred);
    if (m) return min(lo + (uint32_t)__ffs(m) - 1u, hi);
    lo += 32;
  }
  while (lo < hi) {
    const uint32_t span = hi - lo, step = (span + 31u) / 32u;
    const uint32_t cs = lo + lane * step;
    const bool empty = cs >= hi;
    const uint32_t e = empty ? 0u : min(cs + step - 1u, hi - 1u);
    const bool pred = empty || __ldg(last + e) >= dmin;
    const unsigned m = __ballot_sync(0xffffffffu, pred);
    if (!m) return hi;
    const uint32_t fcs = lo + ((uint32_t)__ffs(m) - 1u) * step;
    if (fcs >= hi) return hi;
    lo = fcs; hi = min(fcs + step - 1u, hi - 1u);
  }
  return lo;
}

// Decode block `blk` of a term (full block, or the vint tail when blk == nfull) into docs/tfs[128] and rebuild its
// presence filter.  Every lane calls it; returns the number of postings (docs beyond it are TERMINATED) and the
// last doc through `last`.
// `staged` (nullable): the packed bytes of this block in shared memory, put there ahead of time by the TMA unit.
__device__ uint32_t o3_decode(const SegView& S, const uint4* __restrict__ a128, const OTerm& c, uint32_t blk, uint32_t prev_last,
                              uint32_t* docs, uint32_t* tfs, uint32_t* bloom, uint32_t lane, uint32_t& last, const uint4* staged = nullptr) {
  __syncwarp();
  if (lane < 16) bloom[lane] = 0;
  uint32_t n;
  uint4 d;
  if (blk < c.nfull) {
    const uint32_t idx = c.first + blk;
    const uint32_t bits = S.b_bits[idx], db = bits & 0x3fu, strict = (bits >> 6) & 1u, tb = bits >> 8;
    uint4 f = make_uint4(1, 1, 1, 1);
    if (staged) {
      d = unpack4<true>(staged, db, lane);
      if (S.record >= 1) f = unpack4<true>(staged + db, tb, lane);
    } else {
      const uint4* base = a128 + c.adata + (S.b_off[idx] >> 4);
      d = unpack4(base, db, lane);
      if (S.record >= 1) f = unpack4(base + db, tb, lane);
    }
    if (S.record >= 1) { f.x += strict; f.y += strict; f.z += strict; f.w += strict; }
    d.x += strict; d.y += d.x + strict; d.z += d.y + strict; d.w += d.z + strict;
    const uint32_t incl = warp_scan_incl(d.w, lane);
    const uint32_t before = incl - d.w + ((strict && prev_last == 0) ? 0xFFFFFFFFu : prev_last);  // offset 0 == None
    d.x += before; d.y += before; d.z += before; d.w += before;
    ((uint4*)docs)[lane] = d; ((uint4*)tfs)[lane] = f;
    n = 128;
  } else {
    // vint tail (compression/vint.rs), parsed from the original bytes 32 at a time with a ballot over the stop bits
    n = c.df - c.nfull * 128u;
    const uint8_t* bytes = (const uint8_t*)S.p32 + c.tail_off;
    const uint32_t nbytes = (uint32_t)min((uint64_t)1340, c.end_off - c.tail_off);
    for (uint32_t i = lane; i < 128; i += 32) { docs[i] = 0; tfs[i] = 1; }
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
          if (idx < n) docs[idx] = v; else tfs[idx - n] = v;
        }
      }
      seen += __popc(m);
    }
    __syncwarp();
    d = ((uint4*)docs)[lane];
    d.y += d.x; d.z += d.y; d.w += d.z;
    const uint32_t incl = warp_scan_incl(d.w, lane);
    const uint32_t before = incl - d.w + prev_last;
    d.x += before; d.y += before; d.z += before; d.w += before;
    const uint32_t k0 = lane * 4;
    if (k0 + 0 >= n) d.x = TERMINATED;
    if (k0 + 1 >= n) d.y = TERMINATED;
    if (k0 + 2 >= n) d.z = TERMINATED;
    if (k0 + 3 >= n) d.w = TERMINATED;
    ((uint4*)docs)[lane] = d;
  }
  __syncwarp();  // filter words are zero, the block is in place
  const uint32_t k0 = lane * 4;
  if (k0 + 0 < n) atomicOr(bloom + ((d.x >> 5) & 15u), 1u << (d.x & 31u));
  if (k0 + 1 < n) atomicOr(bloom + ((d.y >> 5) & 15u), 1u << (d.y & 31u));
  if (k0 + 2 < n) atomicOr(bloom + ((d.z >> 5) & 15u), 1u << (d.z & 31u));
  if (k0 + 3 < n) atomicOr(bloom + ((d.w >> 5) & 15u), 1u << (d.w & 31u));
  __syncwarp();
  last = n ? docs[n - 1] : 0u;
  return n;
}

// MODE 1: OR (tantivy weights, query-order f32 sum), MODE 2: Stract BM25 + f64 linear signal combine
// At least 6 resident CTAs per SM caps the registers at 80 (5 would allow 96; 8 would cap them at 64 and spill); the
// kernel is latency-bound, so occupancy is what the choice trades against spills
template <int MODE, int TMAX>
__global__ void __launch_bounds__(WQ * 32, 6) k_or3(const WParams P) {
  static_assert(MODE == 1 || MODE == 2, "k_or3 covers the union modes");
  __shared__ float cache[256];
  __shared__ __align__(16) uint32_t s_docs[WQ][TMAX * 128];
  __shared__ __align__(16) uint32_t s_tfs[WQ][TMAX * 128];
  __shared__ uint32_t s_bloom[WQ][TMAX * 16];
  __shared__ OTerm s_tc[WQ][TMAX];
  __shared__ uint32_t s_misc[WQ][32];
  // TMA staging: while a term's current block is being consumed, the bytes of its NEXT block travel from HBM/L2 into this
  // buffer (one cp.async.bulk per block, completion on the term's mbarrier), so the next refill unpacks from shared
  // memory instead of waiting for two dependent global loads.  Blocks wider than O3_STAGE_BYTES take the direct path.
  __shared__ __align__(16) unsigned char s_stage[WQ][TMAX][O3_STAGE_BYTES];
  __shared__ __align__(8) uint64_t s_bar[WQ][TMAX];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (uint32_t i = threadIdx.x; i < 256; i += WQ * 32) cache[i] = P.cache[i];
  __syncthreads();  // the only block barrier
  const uint32_t item = blockIdx.x * WQ + warp;
  if (item >= P.n_items) return;
  const SegView& S = P.S;
  uint32_t* docs = s_docs[warp]; uint32_t* tfs = s_tfs[warp]; uint32_t* bloom = s_bloom[warp];
  OTerm* tc = s_tc[warp];
  uint32_t* s_rstart = s_misc[warp];        // [TMAX + 1]
  uint32_t* s_pos = s_misc[warp] + 12;      // [TMAX]
  uint32_t* s_count = s_misc[warp] + 24;
  const uint32_t TM = P.n_terms_max;
  const uint32_t q = P.item_q ? P.item_q[item] : item;
  const uint32_t lo_doc = P.item_q ? P.item_lo[item] : 0u, hi_doc = P.item_q ? P.item_hi[item] : 0xFFFFFFFFu;
  const uint32_t oq = P.item_q ? P.item_out[item] : (P.q_orig ? P.q_orig[q] : q);
  const uint32_t T = min(P.q_nterms[q], (uint32_t)TMAX);
  uint64_t* khi = P.g_khi + (size_t)item * P.cap; uint32_t* klo = P.g_klo + (size_t)item * P.cap;
  const bool ranged = lo_doc > 0 || hi_doc != 0xFFFFFFFFu;

  // ---- cursors: lane t owns term t
  uint32_t my_pos = 0, my_len = 0, my_last = 0, my_cur = 0, my_prev = 0;
  bool my_done = true, my_tail_done = false;
  uint32_t my_pf = O3_NONE, my_phase = 0;   // block whose bytes are (being) staged for this lane's term; parity to wait for
  uint64_t* bar = s_bar[warp];
  if (lane < TMAX) mbar_init(bar + lane, 1);
  mbar_fence_init();
  __syncwarp();
  unsigned long long budget = 64;
  if (lane < T) {
    OTerm c;
    const uint32_t ord = P.q_terms[(size_t)q * TM + lane];
    c.first = S.t_first[ord]; c.df = S.t_df[ord]; c.nfull = c.df >> 7;
    c.adata = P.t_aoff[ord]; c.end_off = S.t_end_off[ord];
    c.tail_off = S.t_data_off[ord] + S.b_off[c.first + c.nfull];
    c.weight = P.q_weights[(size_t)q * TM + lane];
    tc[lane] = c;
    my_done = (c.df == 0);
    budget = 4ull * (c.nfull + 2);
  }
  if (lane < TMAX * 16) bloom[lane] = 0;
  if (TMAX * 16 > 32) for (uint32_t i = 32 + lane; i < TMAX * 16; i += 32) bloom[i] = 0;
  if (lane == 0) *s_count = 0;
  for (int o = 16; o; o >>= 1) budget += __shfl_xor_sync(0xffffffffu, budget, o);
  __syncwarp();
  if (lo_doc > 0) {  // start every cursor at the first block that can hold a doc >= lo
    for (uint32_t s = 0; s < T; s++) {
      const OTerm& c = tc[s];
      if (c.nfull == 0) continue;
      const uint32_t j = o3_dir_search(S.b_last + c.first, 0, c.nfull, lo_doc, lane);
      if (lane == s && j > 0) { my_cur = j; my_prev = S.b_last[c.first + j - 1]; }
    }
  }
  bool thr_on = false; uint64_t thr_hi = 0; uint32_t thr_lo = 0;   // warp-uniform
  unsigned long long my_docs = 0, my_blocks = 0;
  bool watchdog = false, bad_doc = false;

  while (T > 0) {
    if (budget-- == 0) { watchdog = true; break; }
    // ---- (1) refill every exhausted cursor (a block that lies entirely below `lo` is consumed at once, so loop)
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
          if (lane < 16) bloom[s * 16 + lane] = 0;   // no current block: nothing can match
          __syncwarp();
          continue;
        }
        uint32_t last;
        const uint4* staged = nullptr;
        const uint32_t pf = __shfl_sync(0xffffffffu, my_pf, s), ph = __shfl_sync(0xffffffffu, my_phase, s);
        if (pf != O3_NONE) {               // an outstanding copy is always waited for before its buffer / barrier is reused
          mbar_wait(bar + s, ph);
          if (pf == cur) staged = (const uint4*)s_stage[warp][s];
          if (lane == (uint32_t)s) { my_pf = O3_NONE; my_phase ^= 1u; }
        }
        const uint32_t n = o3_decode(S, P.a128, c, cur, prev, docs + s * 128, tfs + s * 128, bloom + s * 16, lane, last, staged);
        my_blocks++;
        if (cur + 1 < c.nfull) {  // o3_decode ended with a warp barrier: every lane is done with the staging buffer
          uint32_t issued = 0;
          if (lane == 0) {
            const uint32_t idx = c.first + cur + 1, bits = S.b_bits[idx];
            const uint32_t bytes = ((bits & 0x3fu) + (bits >> 8)) * 16u;
            if (bytes != 0 && bytes <= O3_STAGE_BYTES) {
              mbar_expect_tx(bar + s, bytes);
              tma_load_1d(s_stage[warp][s], P.a128 + c.adata + (S.b_off[idx] >> 4), bytes, bar + s);
              issued = 1;
            }
          }
          issued = __shfl_sync(0xffffffffu, issued, 0);
          if (issued && lane == (uint32_t)s) my_pf = cur + 1;
        }
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
    // ---- (2) bound: every posting <= the smallest last-doc is final
    const bool active = lane < T && !my_done;
    if (!__any_sync(0xffffffffu, active)) break;
    uint32_t bound = __reduce_min_sync(0xffffffffu, active ? my_last : 0xFFFFFFFFu);
    if (ranged && bound >= hi_doc) bound = hi_doc - 1u;
    // ---- (3) this round's slice of every term
    uint32_t rhi = my_pos;
    if (active) rhi = min(lower_bound128(docs + lane * 128, bound + 1u), my_len);
    const uint32_t cnt = rhi - my_pos;
    const uint32_t incl = warp_scan_incl(cnt, lane);
    const uint32_t R = __shfl_sync(0xffffffffu, incl, 31);
    __syncwarp();
    if (lane <= T) s_rstart[lane] = incl - cnt;   // lanes >= T have cnt == 0: s_rstart[T] == R
    if (lane < T) s_pos[lane] = my_pos;
    const uint32_t have = *s_count;   // read before the barrier: behind it other lanes push
    __syncwarp();
    if (have + R > P.cap) {
      w_sort_prefix_desc(khi, klo, have, P.cap, lane);
      const uint32_t c = min(have, P.k);
      if (c == P.k) { thr_on = true; thr_hi = khi[P.k - 1]; thr_lo = klo[P.k - 1]; }
      __syncwarp();
      if (lane == 0) *s_count = c;
      __syncwarp();
    }
    // ---- (4) score.  The global gathers of an entry (fieldnorm byte, 32-B signal row) depend only on its doc id:
    // they are issued for U entries per lane before any is consumed.
    constexpr int U = 2;
    const bool sig4 = (MODE == 2) && P.n_cols == 4;
    for (uint32_t eb = lane; eb < R; eb += 32 * U) {
      uint32_t pi[U], pj[U], pd[U], pf[U]; bool pv[U];
      double2 ps0[U], ps1[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const uint32_t e = eb + 32 * u;
        pv[u] = e < R; pi[u] = 0; pj[u] = 0; pd[u] = 0; pf[u] = 0;
        ps0[u] = make_double2(0.0, 0.0); ps1[u] = make_double2(0.0, 0.0);
        if (pv[u]) {
          uint32_t i = 0;
#pragma unroll
          for (int x = 1; x < TMAX; x++) if ((uint32_t)x < T && e >= s_rstart[x]) i = x;   // s_rstart ascends
          pi[u] = i; pj[u] = s_pos[i] + (e - s_rstart[i]); pd[u] = docs[i * 128 + pj[u]];
          if (pd[u] >= S.max_doc) { pv[u] = false; bad_doc = true; continue; }   // corrupt deltas: never index the doc tables with it
          pf[u] = S.fieldnorm[pd[u]];
          if (sig4) { const double2* r = (const double2*)(P.sig + (size_t)pd[u] * 4); ps0[u] = __ldg(r); ps1[u] = __ldg(r + 1); }
        }
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        if (!pv[u]) continue;
        const uint32_t i = pi[u], d = pd[u];
        const uint32_t bw = (d >> 5) & 15u, bb = 1u << (d & 31u);
        uint32_t tf[TMAX];
        bool owner = true;
#pragma unroll
        for (int x = 0; x < TMAX; x++) {
          tf[x] = 0;
          if ((uint32_t)x >= T || !owner) continue;
          if ((uint32_t)x == i) { tf[x] = tfs[i * 128 + pj[u]]; continue; }
          if (!(bloom[x * 16 + bw] & bb)) continue;                     // certainly not in term x's block
          const uint32_t jj = lower_bound128(docs + x * 128, d);
          if (jj < 128u && docs[x * 128 + jj] == d) {
            if ((uint32_t)x < i) owner = false;                         // a lower slot owns this doc
            else tf[x] = tfs[x * 128 + jj];
          }
        }
        if (!owner) continue;
        my_docs++;
        const float norm = cache[pf[u]];
        uint64_t kh;
        if (MODE == 2) {
          float bm = 0.0f;
#pragma unroll
          for (int x = 0; x < TMAX; x++) if ((uint32_t)x < T) {
            float sc = 0.0f;
            if (tf[x]) { const float t = (float)tf[x]; sc = __fmul_rn(tc[x].weight, __fdiv_rn(__fmul_rn(t, P.k1p1), __fadd_rn(t, norm))); }
            bm = __fadd_rn(bm, sc);
          }
          double total = __dadd_rn(0.0, __dmul_rn(P.coeff_text, (double)bm));
          if (sig4) {
            total = __dadd_rn(total, __dmul_rn(P.coeffs[0], ps0[u].x)); total = __dadd_rn(total, __dmul_rn(P.coeffs[1], ps0[u].y));
            total = __dadd_rn(total, __dmul_rn(P.coeffs[2], ps1[u].x)); total = __dadd_rn(total, __dmul_rn(P.coeffs[3], ps1[u].y));
          } else {
            for (uint32_t c = 0; c < P.n_cols; c++) total = __dadd_rn(total, __dmul_rn(P.coeffs[c], P.sig[(size_t)d * P.n_cols + c]));
          }
          kh = ord_f64(total);
        } else {
          float total = 0.0f;
#pragma unroll
          for (int x = 0; x < TMAX; x++) if ((uint32_t)x < T && tf[x]) {
            const float t = (float)tf[x];
            total = __fadd_rn(total, __fmul_rn(tc[x].weight, __fdiv_rn(t, __fadd_rn(t, norm))));
          }
          kh = (uint64_t)ord_f32(total) << 32;
        }
        const uint32_t kl = ~d;
        if (thr_on && !key_gt(kh, kl, thr_hi, thr_lo)) continue;
        const uint32_t at = atomicAdd(s_count, 1u);
        khi[at] = kh; klo[at] = kl;
      }
    }
    // ---- (5) consume the slice
    if (active) {
      my_pos = rhi;
      if (ranged && my_pos < my_len && docs[lane * 128 + my_pos] >= hi_doc) my_done = true;
    }
    __syncwarp();
  }
  if (my_pf != O3_NONE) mbar_wait(bar + lane, my_phase);   // no copy may still be in flight when the warp leaves
  __threadfence_block();
  __syncwarp();
  w_sort_prefix_desc(khi, klo, *s_count, P.cap, lane);
  const uint32_t n = min(*s_count, P.k);
  for (uint32_t i = lane; i < n; i += 32) {
    P.o_docs[(size_t)oq * P.k + i] = ~klo[i];
    if (MODE == 2) P.o_totals[(size_t)oq * P.k + i] = unord_f64(khi[i]);
    else P.o_scores[(size_t)oq * P.k + i] = unord_f32((uint32_t)(khi[i] >> 32));
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
