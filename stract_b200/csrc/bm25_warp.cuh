// bm25_warp.cuh -- k_topk_warp<MODE>: one WARP per query (4 queries per 128-thread CTA), no block barriers.
//
// Serves the batches k_and3 and k_or3 do not (see the header of bm25.cu): AND with a single-clause query above 65 536
// postings, and the signal combine with max_docs.  Block-synchronous walk of the query terms' posting lists: every
// round takes `bound` = smallest last-doc of the current blocks (every posting <= bound is final), membership is a
// 7-step search in the other terms' decoded blocks, the lowest slot containing a doc owns it, and the exact top-k
// uses a TopNComputer-style threshold (top_score_collector.rs:501-554).  Laid out for throughput on a 10k-query batch:
//   * a warp decodes a 128-doc BitPacker4x block by itself: lane s owns slot s of the four interleaved lane
//     streams, i.e. docs 4s..4s+3; the block bytes are read as 16-byte vectors from a 16-byte aligned copy of the
//     block regions made at segment open (every block is a multiple of 16 bytes), so one LDG.128 returns word w
//     of all four streams; the strict-delta prefix sum is 3 adds + a 5-step warp scan;
//   * per-term state and the decoded blocks live in per-warp shared memory (1 KB per term), so ~32 warps =
//     32 independent queries are resident per SM and hide each other's gather latency -- one CTA per query was
//     bound by barrier and dependent-load latency with only 6 queries per SM;
//   * the 2k-entry candidate buffer lives in global memory (L2): pushes are rare once the threshold is up
//     (~k ln(n/k) per query) and the warp-level bitonic truncation runs a handful of times per query.
#pragma once

namespace sb200 {

constexpr int WQ = 4;  // queries (warps) per CTA

struct WTerm {  // per (warp, term) cursor, warp-uniform values kept in shared memory
  uint64_t adata;      // 16-B aligned block region (in uint4 units) inside the aligned copy
  uint64_t tail_off;   // absolute byte offset of the vint tail in the original file
  uint64_t end_off;
  uint32_t first, nfull, df, cur_blk, len, pos, last_doc, prev_last, done, tail_done;
  float weight;
  uint32_t _pad[3];   // sizeof == 80: keeps the next warp's uint4 arrays 16-byte aligned
};
static_assert(sizeof(WTerm) % 16 == 0, "WTerm must keep 16-byte alignment of the per-warp arrays");

struct WParams {
  SegView S;
  const uint4* a128;            // aligned block regions
  const uint64_t* t_aoff;       // per term: offset of its block region in a128 (uint4 units)
  const uint32_t* q_terms; const uint32_t* q_nterms; const float* q_weights; const float* cache;
  const uint32_t* q_orig;   // slot -> caller's query index (slots are ordered by decreasing work)
  uint32_t n_queries, n_terms_max, k, cap;
  // work items: (query slot, doc range, output slot); null item_q = one item per query over the whole doc space
  uint32_t n_items; const uint32_t* item_q; const uint32_t* item_lo; const uint32_t* item_hi; const uint32_t* item_out;
  float k1p1; double coeff_text; const double* sig; uint32_t n_cols; const double* coeffs; uint32_t max_docs;
  uint64_t* g_khi; uint32_t* g_klo;   // [n_queries][cap] candidate buffers
  uint32_t* o_docs; float* o_scores; double* o_totals; uint32_t* o_n; unsigned long long* counters;
};

__device__ __forceinline__ uint32_t warp_scan_incl(uint32_t x, uint32_t lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const uint32_t n = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += n; }
  return x;
}

// four consecutive values (k = 4*slot .. 4*slot+3) of a 128-value BitPacker4x stream stored at `base` (uint4 units);
// STAGED: `base` points into shared memory (a block the TMA unit copied there), so plain loads instead of ld.global.nc
template <bool STAGED = false>
__device__ __forceinline__ uint4 unpack4(const uint4* __restrict__ base, uint32_t nb, uint32_t slot) {
  if (nb == 0) return make_uint4(0, 0, 0, 0);
  const uint32_t bit = slot * nb, w = bit >> 5, sh = bit & 31u;
  const uint4 lo = STAGED ? base[w] : __ldg(base + w);
  uint4 hi = make_uint4(0, 0, 0, 0);
  if (sh + nb > 32) hi = STAGED ? base[w + 1] : __ldg(base + w + 1);
  const uint32_t mask = nb == 32 ? 0xFFFFFFFFu : ((1u << nb) - 1u);
  return make_uint4(__funnelshift_r(lo.x, hi.x, sh) & mask, __funnelshift_r(lo.y, hi.y, sh) & mask,
                    __funnelshift_r(lo.z, hi.z, sh) & mask, __funnelshift_r(lo.w, hi.w, sh) & mask);
}

// decode the next block of term slot s for this warp; every lane calls it
__device__ void w_decode_next(const WParams& P, WTerm* st, uint32_t* docs_all, uint32_t* tfs_all, int s, uint32_t lane) {
  const SegView& S = P.S;
  WTerm& T = st[s];
  uint32_t* docs = docs_all + s * 128; uint32_t* tfs = tfs_all + s * 128;
  __syncwarp();
  const uint32_t blk = T.cur_blk, prev_last = T.prev_last;
  if (blk < T.nfull) {
    const uint32_t idx = T.first + blk;
    const uint32_t bits = S.b_bits[idx], db = bits & 0x3fu, strict = (bits >> 6) & 1u, tb = bits >> 8;
    const uint4* base = P.a128 + T.adata + (S.b_off[idx] >> 4);
    uint4 d = unpack4(base, db, lane);
    uint4 f = make_uint4(1, 1, 1, 1);
    if (S.record >= 1) { f = unpack4(base + db, tb, lane); f.x += strict; f.y += strict; f.z += strict; f.w += strict; }
    d.x += strict; d.y += d.x + strict; d.z += d.y + strict; d.w += d.z + strict;   // lane-local inclusive sums
    const uint32_t incl = warp_scan_incl(d.w, lane);
    const uint32_t before = incl - d.w + ((strict && prev_last == 0) ? 0xFFFFFFFFu : prev_last);  // offset 0 == None
    d.x += before; d.y += before; d.z += before; d.w += before;
    ((uint4*)docs)[lane] = d; ((uint4*)tfs)[lane] = f;
    const uint32_t last = __shfl_sync(0xffffffffu, d.w, 31);
    __syncwarp();
    if (lane == 0) { T.len = 128; T.pos = 0; T.last_doc = last; T.prev_last = last; T.cur_blk = blk + 1; }
  } else {
    // vint tail (compression/vint.rs): values are runs of bytes ending with the stop bit; parsed from the
    // original bytes 32 at a time with a ballot over the stop bits
    const uint32_t n = T.df - T.nfull * 128u;
    const uint8_t* bytes = (const uint8_t*)S.p32 + T.tail_off;
    const uint32_t nbytes = (uint32_t)min((uint64_t)1340, T.end_off - T.tail_off);
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
    uint4 d = ((uint4*)docs)[lane];
    d.y += d.x; d.z += d.y; d.w += d.z;
    const uint32_t incl = warp_scan_incl(d.w, lane);
    const uint32_t before = incl - d.w + prev_last;
    d.x += before; d.y += before; d.z += before; d.w += before;
    const uint32_t k0 = lane * 4;
    if (k0 + 0 >= n) d.x = TERMINATED; if (k0 + 1 >= n) d.y = TERMINATED; if (k0 + 2 >= n) d.z = TERMINATED; if (k0 + 3 >= n) d.w = TERMINATED;
    ((uint4*)docs)[lane] = d;
    __syncwarp();
    if (lane == 0) { T.len = n; T.pos = 0; T.last_doc = n ? docs[n - 1] : 0; T.prev_last = T.last_doc; T.cur_blk = blk + 1; T.tail_done = 1; }
  }
  __syncwarp();
}

// move term slot s to the first full block (>= its cursor) whose last doc is >= L
__device__ void w_dir_skip(const WParams& P, WTerm* st, int s, uint32_t L, uint32_t lane) {
  __syncwarp();
  const WTerm& t = st[s];
  const uint32_t first = t.first, nfull = t.nfull;
  uint32_t j = nfull;
  for (uint32_t base = t.cur_blk; base < nfull; base += 32) {
    const uint32_t idx = base + lane;
    const bool pred = idx < nfull && __ldg(P.S.b_last + first + idx) >= L;
    const unsigned m = __ballot_sync(0xffffffffu, pred);
    if (m) { j = base + (uint32_t)__ffs(m) - 1u; break; }
  }
  if (lane == 0 && j > st[s].cur_blk) { st[s].cur_blk = j; st[s].prev_last = P.S.b_last[first + j - 1]; }
  __syncwarp();
}

// warp-level bitonic sort (descending) of the query's candidate buffer in global memory
__device__ void w_sort_keys_desc(uint64_t* khi, uint32_t* klo, uint32_t cap, uint32_t lane) {
  for (uint32_t size = 2; size <= cap; size <<= 1) {
    for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
      __syncwarp();
      for (uint32_t i = lane; i < (cap >> 1); i += 32) {
        const uint32_t lo = 2 * i - (i & (stride - 1));
        const uint32_t hi = lo + stride;
        const bool desc = ((lo & size) == 0);
        const uint64_t ah = khi[lo], bh = khi[hi]; const uint32_t al = klo[lo], bl = klo[hi];
        const bool swap = desc ? key_gt(bh, bl, ah, al) : key_gt(ah, al, bh, bl);
        if (swap) { khi[lo] = bh; klo[lo] = bl; khi[hi] = ah; klo[hi] = al; }
      }
    }
  }
  __syncwarp();
}

// sorts the first `count` candidates: only the next power of two is touched (zero keys pad it), the buffer is
// never initialised as a whole -- most AND queries hold a few dozen candidates in a 2048-entry buffer
__device__ __forceinline__ void w_sort_prefix_desc(uint64_t* khi, uint32_t* klo, uint32_t count, uint32_t cap, uint32_t lane) {
  uint32_t n2 = 2; while (n2 < count) n2 <<= 1;
  if (n2 > cap) n2 = cap;
  __syncwarp();
  for (uint32_t i = count + lane; i < n2; i += 32) { khi[i] = 0; klo[i] = 0; }
  w_sort_keys_desc(khi, klo, n2, lane);
}

template <int MODE>
__global__ void __launch_bounds__(WQ * 32) k_topk_warp(const WParams P) {
  static_assert(MODE == 0 || MODE == 2, "k_topk_warp serves AND and the signal combine; OR goes to k_or3");
  SB_DYN_SMEM(smem_raw);
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t TM = P.n_terms_max;
  // layout: cache[256] | per warp: docs[TM][128] tfs[TM][128] st[TM] misc[32]
  float* cache = (float*)smem_raw;
  const size_t per_warp = (size_t)TM * 128 * 8 + sizeof(WTerm) * TM + 32 * 4;
  unsigned char* wp = smem_raw + 1024 + (size_t)warp * per_warp;
  uint32_t* docs = (uint32_t*)wp;
  uint32_t* tfs = docs + TM * 128;
  WTerm* st = (WTerm*)(tfs + TM * 128);
  uint32_t* misc = (uint32_t*)(st + TM);
  uint32_t* s_count = misc + 0;
  uint32_t* s_rstart = misc + 4;   // [MAXT+1]
  uint32_t* s_rhi = misc + 14;     // [MAXT]
  for (uint32_t i = threadIdx.x; i < 256; i += WQ * 32) cache[i] = P.cache[i];
  __syncthreads();  // the only block barrier: the shared norm cache
  // one warp = one work item = (query slot, doc range [lo, hi)); large queries are cut into several items so the
  // batch is not bounded by its largest query, their partial top-k lists are merged by k_merge_topk
  const uint32_t item = blockIdx.x * WQ + warp;
  if (item >= P.n_items) return;
  const SegView& S = P.S;
  const uint32_t q = P.item_q ? P.item_q[item] : item;
  const uint32_t lo_doc = P.item_q ? P.item_lo[item] : 0u, hi_doc = P.item_q ? P.item_hi[item] : 0xFFFFFFFFu;
  const uint32_t oq = P.item_q ? P.item_out[item] : (P.q_orig ? P.q_orig[q] : q);   // output slot
  const uint32_t T = P.q_nterms[q];
  uint64_t* khi = P.g_khi + (size_t)item * P.cap; uint32_t* klo = P.g_klo + (size_t)item * P.cap;
  if (lane < TM) {
    WTerm& t = st[lane];
    t.done = 1; t.len = 0; t.pos = 0; t.df = 0; t.nfull = 0; t.cur_blk = 0; t.tail_done = 0; t.last_doc = 0; t.prev_last = 0;
    if (lane < T) {
      const uint32_t ord = P.q_terms[(size_t)q * TM + lane];
      t.first = S.t_first[ord]; t.df = S.t_df[ord]; t.nfull = t.df >> 7;
      t.adata = P.t_aoff[ord]; t.end_off = S.t_end_off[ord];
      t.tail_off = S.t_data_off[ord] + S.b_off[t.first + t.nfull];
      t.done = (t.df == 0); t.weight = P.q_weights[(size_t)q * TM + lane];
    }
  }
  if (lane == 0) *s_count = 0;
  __syncwarp();
  bool thr_on = false; uint64_t thr_hi = 0; uint32_t thr_lo = 0;   // warp-uniform
  unsigned long long my_docs = 0, my_blocks = 0;
  uint32_t cand_seen = 0;
  unsigned long long budget = 64;
  for (uint32_t s = 0; s < T; s++) budget += 4ull * (st[s].nfull + 2);
  bool watchdog = false, bad_doc = false;
  if (lo_doc > 0)  // start every cursor at the first block that can hold a doc >= lo
    for (uint32_t s = 0; s < T; s++) if (!st[s].done && st[s].nfull) w_dir_skip(P, st, s, lo_doc, lane);
  const bool ranged = lo_doc > 0 || hi_doc != 0xFFFFFFFFu;

  while (T > 0) {
    if (budget-- == 0) { watchdog = true; break; }
    // (1) refill
    for (uint32_t s = 0; s < T; s++) {
      const WTerm& t = st[s];
      if (!t.done && t.pos >= t.len) {
        if (MODE == 0 && T > 1) {
          uint32_t L = 0;
          for (uint32_t x = 0; x < T; x++) { const WTerm& u = st[x]; if (x != s && !u.done && u.pos < u.len) L = max(L, docs[x * 128 + u.pos]); }
          if (L > 0 && t.cur_blk < t.nfull) w_dir_skip(P, st, s, L, lane);
        }
        const bool more = (t.cur_blk < t.nfull) || (t.cur_blk == t.nfull && !t.tail_done && (t.df & 127u));
        if (more) { w_decode_next(P, st, docs, tfs, s, lane); my_blocks++; }
        else { __syncwarp(); if (lane == 0) st[s].done = 1; __syncwarp(); }
      }
    }
    // (1a) clamp to this item's doc range: drop docs below lo, retire a term once its head reaches hi
    if (ranged) {
      __syncwarp();
      if (lane < T) {
        WTerm& w = st[lane];
        if (!w.done && w.pos < w.len) {
          const uint32_t p = lower_bound128(docs + lane * 128, lo_doc);
          if (p > w.pos) w.pos = min(p, w.len);
          if (w.pos < w.len && docs[lane * 128 + w.pos] >= hi_doc) w.done = 1;
        }
      }
      __syncwarp();
      bool again = false;
      for (uint32_t s = 0; s < T; s++) if (!st[s].done && st[s].pos >= st[s].len) again = true;
      if (again) continue;  // a block entirely below lo: refill
    }
    // (1b) AND: decoded blocks entirely below L = max head are dead; so are leading docs below L
    if (MODE == 0 && T > 1) {
      bool alive = true; uint32_t L = 0;
      for (uint32_t s = 0; s < T; s++) { const WTerm& t = st[s]; if (t.done) alive = false; else L = max(L, docs[s * 128 + t.pos]); }
      if (alive) {
        bool dead = false;
        for (uint32_t s = 0; s < T; s++) if (st[s].last_doc < L) dead = true;
        __syncwarp();
        if (lane < T) {
          WTerm& w = st[lane];
          if (w.last_doc < L) { w.pos = 0; w.len = 0; }
          else { const uint32_t p = lower_bound128(docs + lane * 128, L); if (p > w.pos) w.pos = min(p, w.len); }
        }
        __syncwarp();
        if (dead) continue;
      }
    }
    // (2) bound
    uint32_t bound = 0xFFFFFFFFu; bool any = false, all = true;
    for (uint32_t s = 0; s < T; s++) { const WTerm& t = st[s]; if (!t.done) { bound = min(bound, t.last_doc); any = true; } else all = false; }
    if (!any || (MODE == 0 && !all)) break;
    if (ranged && bound >= hi_doc) bound = hi_doc - 1u;
    // (3) ranges
    if (lane < T) {
      const WTerm& t = st[lane];
      uint32_t hi = t.pos;
      if (!t.done) { hi = lower_bound128(docs + lane * 128, bound + 1u); if (hi > t.len) hi = t.len; }
      s_rhi[lane] = hi;
    }
    __syncwarp();
    if (lane == 0) {
      uint32_t acc = 0;
      for (uint32_t s = 0; s < T; s++) { s_rstart[s] = acc; if (MODE != 0 || s == 0) acc += s_rhi[s] - st[s].pos; }
      s_rstart[T] = acc;
    }
    // the fill level is read by every lane BEFORE the barrier: after it other lanes start pushing, and nothing but
    // converged execution would order their atomics behind this read (found by the CPU emulator, tests/emu)
    const uint32_t have = *s_count;
    __syncwarp();
    const uint32_t R = s_rstart[T];
    if (have + R > P.cap) {
      w_sort_prefix_desc(khi, klo, have, P.cap, lane);
      const uint32_t c = min(have, P.k);
      if (c == P.k) { thr_on = true; thr_hi = khi[P.k - 1]; thr_lo = klo[P.k - 1]; }
      __syncwarp();
      if (lane == 0) *s_count = c;
      __syncwarp();
    }
    uint32_t cutoff = 0xFFFFFFFFu; bool last_round = false;
    if (MODE == 2 && P.max_docs) {
      uint32_t mine = 0;
      for (uint32_t e = lane; e < R; e += 32) {
        uint32_t i = 0; while (e >= s_rstart[i + 1]) i++;
        const uint32_t d = docs[i * 128 + st[i].pos + (e - s_rstart[i])];
        bool owner = true;
        for (uint32_t x = 0; x < i && owner; x++) if (!st[x].done) { const uint32_t j = lower_bound128(docs + x * 128, d); if (j < st[x].len && docs[x * 128 + j] == d) owner = false; }
        mine += owner;
      }
      const uint32_t total_owners = __shfl_sync(0xffffffffu, warp_scan_incl(mine, lane), 31);
      if (cand_seen + total_owners >= P.max_docs) {
        last_round = true;
        const uint32_t remaining = P.max_docs - cand_seen;
        uint32_t lo = 0, hi = bound;
        while (lo < hi) {  // smallest doc value v with #owners(doc <= v) >= remaining
          const uint32_t mid = lo + ((hi - lo) >> 1);
          uint32_t c = 0;
          for (uint32_t e = lane; e < R; e += 32) {
            uint32_t i = 0; while (e >= s_rstart[i + 1]) i++;
            const uint32_t d = docs[i * 128 + st[i].pos + (e - s_rstart[i])];
            if (d > mid) continue;
            bool owner = true;
            for (uint32_t x = 0; x < i && owner; x++) if (!st[x].done) { const uint32_t j = lower_bound128(docs + x * 128, d); if (j < st[x].len && docs[x * 128 + j] == d) owner = false; }
            c += owner;
          }
          const uint32_t tot = __shfl_sync(0xffffffffu, warp_scan_incl(c, lane), 31);
          if (tot >= remaining) hi = mid; else lo = mid + 1;
        }
        cutoff = lo;
      }
      cand_seen += total_owners;
    }
    // (4) score.  The global gathers of an entry (fieldnorm byte, 32-B signal row) depend only on its doc id, so
    // they are issued for U entries per lane before any is consumed: U dependent DRAM round trips become one.
    constexpr int U = (MODE == 2) ? 2 : 4;
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
          uint32_t i = 0; while (e >= s_rstart[i + 1]) i++;
          pi[u] = i; pj[u] = st[i].pos + (e - s_rstart[i]); pd[u] = docs[i * 128 + pj[u]];
          pv[u] = pd[u] <= cutoff;
          if (pv[u] && pd[u] >= S.max_doc) { pv[u] = false; bad_doc = true; }  // corrupt deltas: never index the doc tables with it
          if (pv[u]) {
            if (MODE != 0) pf[u] = S.fieldnorm[pd[u]];   // AND: almost every entry fails the membership test, fetch later
            if (sig4) { const double2* r = (const double2*)(P.sig + (size_t)pd[u] * 4); ps0[u] = __ldg(r); ps1[u] = __ldg(r + 1); }
          }
        }
      }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (!pv[u]) continue;
      const uint32_t i = pi[u], j = pj[u], d = pd[u];
      uint32_t fid = pf[u];
      uint32_t tf[MAXT];
      bool ok = true;
#pragma unroll
      for (uint32_t x = 0; x < MAXT; x++) {
        tf[x] = 0;
        if (x >= T || !ok) continue;
        if (x == i) { tf[x] = tfs[i * 128 + j]; continue; }
        bool found = false;
        if (!st[x].done) {
          const uint32_t jj = lower_bound128(docs + x * 128, d);
          if (jj < st[x].len && docs[x * 128 + jj] == d) { found = true; tf[x] = tfs[x * 128 + jj]; }
        }
        if (MODE == 0) { if (!found) ok = false; }
        else if (found && x < i) ok = false;
      }
      if (!ok) continue;
      my_docs++;
      if (MODE == 0) fid = S.fieldnorm[d];
      const float norm = cache[fid];
      uint64_t kh;
      if (MODE == 2) {
        float bm = 0.0f;
#pragma unroll
        for (uint32_t x = 0; x < MAXT; x++) if (x < T) {
          float sc = 0.0f;
          if (tf[x]) { const float t = (float)tf[x]; sc = __fmul_rn(st[x].weight, __fdiv_rn(__fmul_rn(t, P.k1p1), __fadd_rn(t, norm))); }
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
        float sc[MAXT];
#pragma unroll
        for (uint32_t x = 0; x < MAXT; x++) { sc[x] = 0.0f; if (x < T && tf[x]) { const float t = (float)tf[x]; sc[x] = __fmul_rn(st[x].weight, __fdiv_rn(t, __fadd_rn(t, norm))); } }
        float total;
        if (MODE == 0) {
          if (T == 1) total = sc[0];
          else {
            float others = 0.0f;
#pragma unroll
            for (uint32_t x = 2; x < MAXT; x++) if (x < T) others = __fadd_rn(others, sc[x]);
            total = __fadd_rn(__fadd_rn(sc[0], sc[1]), others);
          }
        } else {
          total = 0.0f;
#pragma unroll
          for (uint32_t x = 0; x < MAXT; x++) if (x < T && tf[x]) total = __fadd_rn(total, sc[x]);
        }
        kh = (uint64_t)ord_f32(total) << 32;
      }
      const uint32_t kl = ~d;
      if (thr_on && !key_gt(kh, kl, thr_hi, thr_lo)) continue;
      const uint32_t at = atomicAdd(s_count, 1u);
      khi[at] = kh; klo[at] = kl;
    }
    }
    __syncwarp();
    if (lane < T && !st[lane].done) st[lane].pos = s_rhi[lane];
    __syncwarp();
    if (last_round) break;
  }
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
  if (__any_sync(0xffffffffu, bad_doc)) watchdog = true;   // a decoded doc id outside the segment: reported like a decode failure
  if (lane == 0) {
    if (my_docs) atomicAdd(P.counters + 0, my_docs);
    if (my_blocks) atomicAdd(P.counters + 1, my_blocks);
    if (watchdog) atomicAdd(P.counters + 2, 1ull);
  }
}

// Merge of the partial top-k lists of a query that was cut into several doc-range items (TopCollector::merge_fruits,
// tantivy/src/collector/top_collector.rs:109-129, is the same operation across segments): one CTA per such query,
// all candidates (<= W*k <= 16384) sorted in shared memory with the same (score desc, doc asc) keys.
template <int MODE>
__global__ void __launch_bounds__(256) k_merge_topk(const MergeJob* __restrict__ jobs, uint32_t k, uint32_t capm,
                                                    uint32_t* o_docs, float* o_scores, double* o_totals, uint32_t* o_n) {
  SB_DYN_SMEM(smem_raw);
  uint64_t* khi = (uint64_t*)smem_raw;
  uint32_t* klo = (uint32_t*)(khi + capm);
  const MergeJob job = jobs[blockIdx.x];
  const uint32_t tid = threadIdx.x;
  uint32_t base = 0;
  for (uint32_t s = 0; s < job.n_slots; s++) {
    const uint32_t slot = job.first_slot + s, n = o_n[slot];
    for (uint32_t i = tid; i < n; i += 256) {
      const uint32_t d = o_docs[(size_t)slot * k + i];
      khi[base + i] = (MODE == 2) ? ord_f64(o_totals[(size_t)slot * k + i]) : ((uint64_t)ord_f32(o_scores[(size_t)slot * k + i]) << 32);
      klo[base + i] = ~d;
    }
    base += n;
  }
  // only the next power of two above the entries actually present is padded and sorted (capm = W_max * k is the
  // worst case; most jobs merge a few short lists)
  uint32_t n2 = 2; while (n2 < base) n2 <<= 1;
  if (n2 > capm) n2 = capm;
  for (uint32_t i = base + tid; i < n2; i += 256) { khi[i] = 0; klo[i] = 0; }
  for (uint32_t size = 2; size <= n2; size <<= 1) {
    for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (uint32_t i = tid; i < (n2 >> 1); i += 256) {
        const uint32_t lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
        const bool desc = ((lo & size) == 0);
        const uint64_t ah = khi[lo], bh = khi[hi]; const uint32_t al = klo[lo], bl = klo[hi];
        const bool swap = desc ? key_gt(bh, bl, ah, al) : key_gt(ah, al, bh, bl);
        if (swap) { khi[lo] = bh; klo[lo] = bl; khi[hi] = ah; klo[hi] = al; }
      }
    }
  }
  __syncthreads();
  const uint32_t n = min(base, k);
  for (uint32_t i = tid; i < n; i += 256) {
    o_docs[(size_t)job.out_slot * k + i] = ~klo[i];
    if (MODE == 2) o_totals[(size_t)job.out_slot * k + i] = unord_f64(khi[i]);
    else o_scores[(size_t)job.out_slot * k + i] = unord_f32((uint32_t)(khi[i] >> 32));
  }
  if (tid == 0) o_n[job.out_slot] = n;
}

// copies every term's block region into a 16-byte aligned buffer (one warp per term, byte realignment by funnel shift)
__global__ void k_align_blocks(const uint32_t* __restrict__ p32, const uint64_t* __restrict__ t_data_off,
                               const uint32_t* __restrict__ t_first, const uint32_t* __restrict__ t_df,
                               const uint32_t* __restrict__ b_off, const uint64_t* __restrict__ t_aoff, uint32_t n_terms,
                               uint32_t* dst32) {
  const uint32_t t = (blockIdx.x * (uint32_t)blockDim.x + threadIdx.x) >> 5;
  if (t >= n_terms) return;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t nfull = t_df[t] >> 7;
  const uint32_t nbytes = b_off[t_first[t] + nfull];
  const uint64_t src = t_data_off[t];
  const uint64_t w0 = src >> 2; const uint32_t sh = (uint32_t)(src & 3u) * 8u;
  uint32_t* d = dst32 + t_aoff[t] * 4;
  for (uint32_t w = lane; w < (nbytes >> 2); w += 32) d[w] = __funnelshift_r(__ldg(p32 + w0 + w), __ldg(p32 + w0 + w + 1), sh);
}
__global__ void k_block_units(const uint32_t* __restrict__ t_first, const uint32_t* __restrict__ t_df,
                              const uint32_t* __restrict__ b_off, uint32_t n_terms, uint64_t* units) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n_terms) units[t] = (uint64_t)(b_off[t_first[t] + (t_df[t] >> 7)] >> 4);  // block bytes are multiples of 16
}

}  // namespace sb200
