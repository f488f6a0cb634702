// bm25_phrase.cuh -- phrase queries: PhraseWeight -> PhraseScorer -> TopNComputer (tantivy/src/query/phrase_query).
//
// Positions in HBM (sb200_segment_attach_positions): the field's `.pos` file byte for byte, plus two directories built on the
// device -- per positions block of every term its bit width and byte offset (reader.rs:67-102), and per posting block the
// position offset of its first posting (prefix of the skip entries' tf sums, skip.rs:219,261-266; the vint tail's entry is
// the total of the full blocks).  Blocks are read with funnel-shifted 32-bit loads, so no aligned copy is kept.
//
// A batch runs in three kernels per group of queries:
//   k_phrase_cand    the AND of the phrase's terms with k_and3's machinery (one warp per few blocks of the rarest term,
//                    directory search in the others, Intersection's doc_freq order).  Instead of a score a hit records,
//                    for every term, tf and the position offset of its posting (segment_postings.rs:233-254: the block's
//                    base plus the tfs before the posting in its block).  Capacity df(rarest) per query: no overflow path.
//   k_phrase_verify  one warp per candidate: decodes exactly the deltas [offset, offset + tf) of every term, prefix-sums
//                    them from max_offset - offset (phrase_scorer.rs:371-383), then
//                      slop 0: the count of positions common to all shifted lists (order-free: lane-parallel binary
//                              searches and a warp sum);
//                      slop > 0: lane 0 replays compute_phrase_match / compute_phrase_count / phrase_exists
//                              (phrase_scorer.rs:422-505) in docset order, u8 slops and "finish rest" tail included.
//                    Lists live in shared memory; a candidate whose lists (or carrying-slop buffers) do not fit goes to a
//                    pass over global scratch sized from the first pass's totals.  The carrying-slop merge of >= 3 terms is
//                    not bounded by its inputs (up to ~slop+3 entries per input position and step, compounding over the
//                    steps): while it overflows, the next pass gives it buffers of max(4x, the length it asked for).  Limits:
//                    8 such passes and 2^32 entries per buffer, beyond which the batch fails with SB200_ENOMEM.
//   k_and3_select    exact top-k of the matches by (score desc, doc asc).
#pragma once

namespace sb200 {

constexpr int PH_WARPS = 4;                  // candidates (warps) per CTA of k_phrase_verify
constexpr uint32_t PH_SMEM_WORDS = 1536;     // per-warp position buffer in shared memory

struct PosView {
  const uint32_t* f32;                       // the positions file as words (+64 zero bytes)
  const uint64_t *data_off, *tail_off, *end_off, *count;   // per term
  const uint32_t *first, *nblk;              // per term: first block slot, bit-packed blocks
  const uint64_t* b_off; const uint8_t* b_w; // per block: byte offset from data_off (a term's blocks may pass 4 GiB), bit width
};

// 4 bytes of the file at any byte offset
__device__ __forceinline__ uint32_t ph_word(const uint32_t* f32, uint64_t byte) {
  const uint64_t w = byte >> 2; const uint32_t sh = (uint32_t)(byte & 3u) * 8u;
  return __funnelshift_r(__ldg(f32 + w), __ldg(f32 + w + 1), sh);
}

// value k of a 128-value BitPacker4x block at byte `base` (compress_block_unsorted: no delta)
__device__ __forceinline__ uint32_t ph_unpack_at(const uint32_t* f32, uint64_t base, uint32_t nb, uint32_t k) {
  if (nb == 0) return 0;
  const uint32_t l4 = k & 3u, bit = (k >> 2) * nb, w = bit >> 5, sh = bit & 31u;
  const uint32_t lo = ph_word(f32, base + (uint64_t)(w * 4 + l4) * 4);
  const uint32_t hi = (sh + nb > 32) ? ph_word(f32, base + (uint64_t)((w + 1) * 4 + l4) * 4) : 0u;
  const uint32_t v = __funnelshift_r(lo, hi, sh);
  return nb == 32 ? v : (v & ((1u << nb) - 1u));
}

// the vint tail of term `ord` (uncompress_vint_unsorted_until_end) into tb[0..128); the warp calls it together
__device__ void ph_decode_tail(const PosView& V, uint32_t ord, uint32_t* tb, uint32_t lane) {
  const uint8_t* bytes = (const uint8_t*)V.f32;
  const uint64_t a = V.tail_off[ord];
  const uint32_t nbytes = (uint32_t)(V.end_off[ord] - a);   // attach checked: <= 127 values, ends on a stop byte
  __syncwarp();
  uint32_t seen = 0;
  for (uint32_t base = 0; base < nbytes; base += 32) {
    const uint32_t b = base + lane;
    const uint32_t byte = (b < nbytes) ? bytes[a + b] : 0u;
    const bool stop = (byte & 0x80u) != 0;
    const unsigned m = __ballot_sync(0xffffffffu, stop);
    if (stop) {
      const uint32_t idx = seen + __popc(m & ((1u << lane) - 1u));
      uint32_t v = byte & 0x7Fu, start = b;
      while (start > 0 && b - start < 4 && !(bytes[a + start - 1] & 0x80u)) { start--; v = (v << 7) | (bytes[a + start] & 0x7Fu); }
      if (idx < 128) tb[idx] = v;
    }
    seen += __popc(m);
  }
  __syncwarp();
}

// position deltas [o, o + n) of term `ord` into out[0..n) (shared or global); returns the bytes of the blocks / tail read
__device__ uint64_t ph_read_deltas(const PosView& V, uint32_t ord, uint64_t o, uint32_t n, uint32_t* out, uint32_t* tb, uint32_t lane) {
  const uint32_t nb = V.nblk[ord], first = V.first[ord];
  const uint64_t data = V.data_off[ord], full = (uint64_t)nb * 128u;
  uint64_t bytes = 0;
  if (n && o < full) {
    const uint64_t hi = min(o + n, full);
    for (uint64_t i = o + lane; i < hi; i += 32) {
      const uint32_t b = (uint32_t)(i >> 7);
      out[i - o] = ph_unpack_at(V.f32, data + V.b_off[first + b], V.b_w[first + b], (uint32_t)(i & 127u));
    }
    for (uint32_t b = (uint32_t)(o >> 7); b <= (uint32_t)((hi - 1) >> 7); b++) bytes += (uint64_t)V.b_w[first + b] * 16u;
  }
  if (o + n > full) {
    ph_decode_tail(V, ord, tb, lane);
    for (uint64_t i = max(o, full) + lane; i < o + n; i += 32) out[i - o] = tb[i - full];
    bytes += V.end_off[ord] - V.tail_off[ord];
  }
  __syncwarp();
  return bytes;
}

// positions_with_offset: a[i] = shift + a[0] + ... + a[i] (u32, wrapping like the reference's release build)
__device__ void ph_prefix(uint32_t* a, uint32_t n, uint32_t shift, uint32_t lane) {
  uint32_t carry = shift;
  for (uint32_t base = 0; base < n; base += 32) {
    const uint32_t i = base + lane;
    const uint32_t incl = warp_scan_incl(i < n ? a[i] : 0u, lane);
    if (i < n) a[i] = carry + incl;
    carry += __shfl_sync(0xffffffffu, incl, 31);
  }
  __syncwarp();
}

__device__ __forceinline__ bool ph_contains(const uint32_t* a, uint32_t n, uint32_t x) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (a[mid] < x) lo = mid + 1; else hi = mid; }
  return lo < n && a[lo] == x;
}

__device__ __forceinline__ uint32_t ph_absdiff(uint32_t a, uint32_t b) { return a > b ? a - b : b - a; }

// intersection_count_with_slop(.., update_left = false), phrase_scorer.rs:145-191
__device__ uint32_t ph_count_slop(const uint32_t* l, uint32_t ln, const uint32_t* r, uint32_t rn, uint32_t slop) {
  uint32_t li = 0, ri = 0, count = 0;
  while (li < ln && ri < rn) {
    const uint32_t lv = l[li], rv = r[ri];
    if (ph_absdiff(lv, rv) <= slop) {
      while (li + 1 < ln && l[li + 1] <= rv) li++;
      count++; li++; ri++;
    } else if (lv < rv) li++;
    else ri++;
  }
  return count;
}

// intersection_exists_with_slop, phrase_scorer.rs:193-215
__device__ bool ph_exists_slop(const uint32_t* l, uint32_t ln, const uint32_t* r, uint32_t rn, uint32_t slop) {
  uint32_t li = 0, ri = 0;
  while (li < ln && ri < rn) {
    const uint32_t lv = l[li], rv = r[ri];
    if (ph_absdiff(lv, rv) <= slop) return true;
    if (lv < rv) li++; else ri++;
  }
  return false;
}

// intersection_count_with_carrying_slop, phrase_scorer.rs:232-345.  Left = (lp, ls) with llen positions and lslen slops (0:
// the cleared vector, every slop so far 0); the merged list is built in (pb, sb) of capacity `cap` and swapped in when
// update.  *ovf is set when it does not fit; C.need then holds (an upper bound of) the length the merge wanted.
struct PhCarry { uint32_t *lp, *ls, *pb, *sb; uint32_t llen, lslen, cap; uint64_t need; };
__device__ uint32_t ph_carry(PhCarry& C, const uint32_t* rp, uint32_t rlen, uint32_t max_slop, bool update, bool* ovf) {
  if (C.llen == 0 || rlen == 0) { if (update) { C.llen = 0; C.lslen = 0; } return 0; }
  uint32_t li = 0, ri = 0, count = 0, plen = 0;
  uint64_t extra = 0;
  auto add = [&](uint32_t slop, uint32_t v) {
    if (!update) return;
    const uint8_t s8 = (uint8_t)slop;
    if (plen && C.pb[plen - 1] == v) { if (s8 < C.sb[plen - 1]) C.sb[plen - 1] = s8; }
    else if (plen < C.cap) { C.pb[plen] = v; C.sb[plen] = s8; plen++; }
    else { *ovf = true; extra++; }
  };
  for (;;) {
    const uint32_t lv = C.lp[li], rv = rp[ri];
    const uint32_t sso = li < C.lslen ? C.ls[li] : 0u;
    const uint32_t dist = sso + ph_absdiff(lv, rv);
    if (dist <= max_slop) {
      const bool lsm = lv < rv;
      const uint32_t larger = lsm ? rv : lv;
      const uint32_t* sp = lsm ? C.lp : rp; const uint32_t sn = lsm ? C.llen : rlen;
      uint32_t si = lsm ? li : ri;
      uint32_t new_slop = dist;
      add(new_slop, lsm ? lv : rv);
      while (si + 1 < sn) {
        const uint32_t nv = sp[si + 1];
        if (nv > larger) break;
        si++;
        new_slop = sso + ph_absdiff(nv, larger);
        add(new_slop, nv);
      }
      add(new_slop, larger);
      count++; li++; ri++;
    } else if (lv < rv) li++;
    else ri++;
    if (li >= C.llen || ri >= rlen) {   // finish rest
      if (li >= C.llen) {
        const uint32_t lv2 = C.lp[C.llen - 1], s2 = C.lslen ? C.ls[C.lslen - 1] : 0u;
        for (uint32_t r = ri; r < rlen; r++) { const uint32_t ns = ph_absdiff(lv2, rp[r]) + s2; if (ns <= max_slop) add(ns, rp[r]); }
      } else {
        const uint32_t rv2 = rp[rlen - 1];
        for (uint32_t l = li; l < C.llen; l++) { const uint32_t s2 = l < C.lslen ? C.ls[l] : 0u; const uint32_t ns = ph_absdiff(C.lp[l], rv2) + s2; if (ns <= max_slop) add(ns, C.lp[l]); }
      }
      break;
    }
  }
  if (extra && (uint64_t)plen + extra > C.need) C.need = (uint64_t)plen + extra;
  if (update) {
    uint32_t* t = C.lp; C.lp = C.pb; C.pb = t;
    t = C.ls; C.ls = C.sb; C.sb = t;
    C.llen = plen; C.lslen = plen;
  }
  return count;
}

// ------------------------------------------------------------------ candidates --------------------------------------------
struct PhCandParams {
  A3Params A;                  // segment view, per-slot terms in docset order, units, candidate offsets / counts, counters
  const uint64_t* pos_base;    // per posting block slot (t_first layout): position offset of its first posting
  uint32_t nt;                 // row width of the candidate records
  uint32_t* c_doc; uint64_t* c_off; uint32_t* c_tf;   // [entry], [entry][nt], [entry][nt]
};

// dynamic shared memory: [A3_WARPS][nt][128] u64 position offsets, then [A3_WARPS][nt][128] u32 tfs.  MIN_T: rows with
// fewer terms produce nothing (phrases: 2; optic patterns, bm25_pattern.cuh: 1, every posting of a one-term row is a candidate)
template <uint32_t MIN_T>
__global__ void __launch_bounds__(A3_WARPS * 32) k_phrase_cand(const PhCandParams C) {
  SB_DYN_SMEM(smem_raw);
  __shared__ __align__(16) uint32_t s_docs[A3_WARPS][128];
  __shared__ __align__(16) uint32_t s_tfs[A3_WARPS][128];
  __shared__ __align__(16) uint32_t s_pre[A3_WARPS][128];
  __shared__ uint32_t s_cur[A3_WARPS][MAXT];
  const A3Params& P = C.A;
  const SegView& S = P.S;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t u = blockIdx.x * A3_WARPS + warp;
  if (u >= P.n_units) return;
  uint64_t* r_off = (uint64_t*)smem_raw + (size_t)warp * C.nt * 128;
  uint32_t* r_tf = (uint32_t*)((uint64_t*)smem_raw + (size_t)A3_WARPS * C.nt * 128) + (size_t)warp * C.nt * 128;
  const AUnit U = P.units[u];
  const uint32_t q = U.q, T = P.q_nterms[q];
  uint32_t* sd = s_docs[warp]; uint32_t* stf = s_tfs[warp]; uint32_t* spre = s_pre[warp]; uint32_t* cur = s_cur[warp];
  if (lane < MAXT) cur[lane] = 0;
  __syncwarp();
  if (T < MIN_T) return;
  const A3Term tA = a3_load_term(P, q, 0);
  unsigned long long n_blocks = 0, n_hits = 0;
  bool watchdog = false, bad_doc = false;

  for (uint32_t ablk = U.blk_lo; ablk < U.blk_hi; ablk++) {
    uint32_t d[4], tfa[4];
    uint32_t nA = 128;
    if (ablk < tA.nfull) {
      A3Blk BA;
      const uint4 v = a3_decode_docs(P, tA, ablk, lane, BA);
      const uint4 f = unpack4(BA.base + BA.db, BA.tb, lane);
      d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
      tfa[0] = f.x + BA.strict; tfa[1] = f.y + BA.strict; tfa[2] = f.z + BA.strict; tfa[3] = f.w + BA.strict;
    } else {
      nA = a3_decode_tail(P, tA, sd, stf, lane);
      const uint4 v = ((const uint4*)sd)[lane], f = ((const uint4*)stf)[lane];
      d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
      tfa[0] = f.x; tfa[1] = f.y; tfa[2] = f.z; tfa[3] = f.w;
      __syncwarp();
    }
    n_blocks++;
    {   // position offsets of the A postings: block base + tfs before the posting
      const uint32_t loc = tfa[0] + tfa[1] + tfa[2] + tfa[3];
      uint32_t ex = warp_scan_incl(loc, lane) - loc;
      const uint64_t base = C.pos_base[tA.first + ablk];
#pragma unroll
      for (int b = 0; b < 4; b++) { r_off[lane * 4 + b] = base + ex; r_tf[lane * 4 + b] = tfa[b]; ex += tfa[b]; }
    }
    uint32_t alive = 0;
#pragma unroll
    for (int b = 0; b < 4; b++) if (lane * 4 + b < nA) {
      if (d[b] < S.max_doc) alive |= 1u << b;
      else bad_doc = true;
    }

    for (uint32_t x = 1; x < T; x++) {
      if (!__any_sync(0xffffffffu, alive != 0)) break;
      const A3Term tX = a3_load_term(P, q, x);
      uint32_t pend = alive;
      for (uint32_t guard = 0;; guard++) {
        if (guard > 130u) { watchdog = true; break; }
        uint32_t m = 0xFFFFFFFFu;
#pragma unroll
        for (int b = 3; b >= 0; b--) if ((pend >> b) & 1u) m = d[b];
#pragma unroll
        for (int o = 16; o; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (m == 0xFFFFFFFFu) break;
        const uint32_t jb = a3_dir_search(S, tX, cur[x], m, lane);
        __syncwarp();
        if (lane == 0) cur[x] = jb;
        uint32_t lastB, lenB; bool x_tail = false;
        if (jb < tX.nfull) {
          A3Blk BX;
          const uint4 v = a3_decode_docs(P, tX, jb, lane, BX);
          uint4 f = unpack4(BX.base + BX.db, BX.tb, lane);
          f.x += BX.strict; f.y += BX.strict; f.z += BX.strict; f.w += BX.strict;
          const uint32_t loc = f.x + f.y + f.z + f.w;
          const uint32_t ex = warp_scan_incl(loc, lane) - loc;
          __syncwarp();                       // every lane is done with the previous contents of sd / stf / spre
          ((uint4*)sd)[lane] = v; ((uint4*)stf)[lane] = f;
          ((uint4*)spre)[lane] = make_uint4(ex, ex + f.x, ex + f.x + f.y, ex + f.x + f.y + f.z);
          lastB = __shfl_sync(0xffffffffu, v.w, 31); lenB = 128;
          __syncwarp();
        } else {
          x_tail = true; lastB = 0xFFFFFFFFu;
          lenB = (tX.df & 127u) ? a3_decode_tail(P, tX, sd, stf, lane) : 0u;
          const uint4 f = ((const uint4*)stf)[lane];
          const uint32_t loc = f.x + f.y + f.z + f.w;
          const uint32_t ex = warp_scan_incl(loc, lane) - loc;
          __syncwarp();
          ((uint4*)spre)[lane] = make_uint4(ex, ex + f.x, ex + f.x + f.y, ex + f.x + f.y + f.z);
          __syncwarp();
        }
        const uint64_t xbase = C.pos_base[tX.first + (x_tail ? tX.nfull : jb)];
        n_blocks++;
#pragma unroll
        for (int b = 0; b < 4; b++) {
          if (((pend >> b) & 1u) && d[b] <= lastB) {
            pend &= ~(1u << b);
            bool found = false; uint32_t j = 0;
            if (lenB) { j = lower_bound128(sd, d[b]); found = j < lenB && sd[j] == d[b]; }
            if (!found) alive &= ~(1u << b);
            else { r_off[x * 128 + lane * 4 + b] = xbase + spre[j]; r_tf[x * 128 + lane * 4 + b] = stf[j]; }
          }
        }
        if (x_tail) break;
      }
    }
    // append the candidates with their per-term (position offset, tf)
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
        C.c_doc[pos] = d[b];
        for (uint32_t t = 0; t < T; t++) {
          C.c_off[pos * C.nt + t] = r_off[t * 128 + lane * 4 + b];
          C.c_tf[pos * C.nt + t] = r_tf[t * 128 + lane * 4 + b];
        }
        pos++;
      }
      n_hits += total;
    }
    __syncwarp();
  }
  if (__any_sync(0xffffffffu, bad_doc)) watchdog = true;
  if (lane == 0) {
    if (n_hits) atomicAdd(P.counters + 0, n_hits);
    if (watchdog) atomicAdd(P.counters + 2, 1ull);
  }
}

// ------------------------------------------------------------------ verification ------------------------------------------
struct PhParams {
  PosView V;
  const uint8_t* fieldnorm; const float* cache;
  const uint32_t *q_terms, *q_shift, *q_nterms, *q_slop; const float* q_weight;   // per query slot, terms in docset order
  uint32_t nt; int scoring;
  const uint64_t* cand_off;    // per query slot: start of its candidate records
  const uint64_t* cand_pre;    // [n_slots + 1] prefix of the group's candidate counts
  uint32_t slot0, n_slots;
  const uint32_t* c_doc; const uint64_t* c_off; const uint32_t* c_tf;
  const unsigned long long* list; unsigned long long n;   // list == NULL: candidates 0..n of the group
  uint32_t* scratch; uint32_t factor;                     // scratch == NULL: shared-memory pass (factor 1)
  unsigned long long* scratch_cursor;
  unsigned long long* ov_list; unsigned long long* ov;    // candidates for the next pass; ov[0] = count, ov[1] = their tf sum,
                                                          // ov[3] = the largest merge length / tf sum they asked for
  uint32_t* m_cnt; uint32_t* m_key; uint32_t* m_doc;      // matches, at cand_off[slot]
  unsigned long long* counters;  // [0] candidates [1] matches [2] format errors [3] positions decoded [4] position bytes
                                 // [5] candidates whose merge buffers would exceed 2^32 entries
};

__global__ void __launch_bounds__(PH_WARPS * 32) k_phrase_verify(const PhParams P) {
  __shared__ __align__(16) uint32_t s_buf[PH_WARPS][PH_SMEM_WORDS];
  __shared__ uint32_t s_tail[PH_WARPS][128];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned long long n_match = 0, n_dec = 0, n_bytes = 0;
  bool bad = false;
  for (unsigned long long it = (unsigned long long)blockIdx.x * PH_WARPS + warp; it < P.n; it += (unsigned long long)gridDim.x * PH_WARPS) {
    const unsigned long long c = P.list ? P.list[it] : it;
    uint32_t lo = 0, hi = P.n_slots;   // the slot s with cand_pre[s] <= c < cand_pre[s + 1]
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (P.cand_pre[mid] <= c) lo = mid; else hi = mid; }
    const uint32_t slot = P.slot0 + lo;
    const uint64_t e = P.cand_off[slot] + (c - P.cand_pre[lo]);
    const uint32_t T = P.q_nterms[slot], slop = P.q_slop[slot];
    uint32_t tf[MAXT], st[MAXT];
    uint64_t S = 0;
    for (uint32_t t = 0; t < T; t++) { tf[t] = P.c_tf[e * P.nt + t]; st[t] = (uint32_t)S; S += tf[t]; }
    const bool carry = slop > 0 && T > 2;
    const uint64_t W = carry ? S * P.factor : 0;          // capacity of each carrying-slop buffer
    const uint64_t need = S + 4 * W;
    if (W > 0xFFFFFFFFull) { if (lane == 0) atomicAdd(P.counters + 5, 1ull); continue; }
    uint32_t* buf;
    if (!P.scratch) {
      if (need > PH_SMEM_WORDS) {
        if (lane == 0) { const unsigned long long i = atomicAdd(P.ov + 0, 1ull); P.ov_list[i] = c; atomicAdd(P.ov + 1, (unsigned long long)S); }
        continue;
      }
      buf = s_buf[warp];
    } else {
      unsigned long long off = 0;
      if (lane == 0) off = atomicAdd(P.scratch_cursor, (unsigned long long)need);
      buf = P.scratch + __shfl_sync(0xffffffffu, off, 0);
    }
    bool ok = true;
    uint64_t cand_bytes = 0;
    for (uint32_t t = 0; t < T; t++) {
      const uint32_t ord = P.q_terms[(size_t)slot * P.nt + t];
      const uint64_t o = P.c_off[e * P.nt + t];
      if (o + tf[t] > P.V.count[ord]) { ok = false; break; }   // the skip entries' tf sums disagree with the positions file
      cand_bytes += ph_read_deltas(P.V, ord, o, tf[t], buf + st[t], s_tail[warp], lane);
      ph_prefix(buf + st[t], tf[t], P.q_shift[(size_t)slot * P.nt + t], lane);
    }
    if (!ok) { bad = true; continue; }
    uint32_t count = 0; bool match = false;
    if (slop == 0) {   // |L0 n L1 n ... n L(T-1)|: intersection + intersection_count (phrase_scorer.rs:82-136,496)
      uint32_t mine = 0;
      for (uint32_t i = lane; i < tf[0]; i += 32) {
        const uint32_t x = buf[i];
        bool all = true;
        for (uint32_t t = 1; t < T && all; t++) all = ph_contains(buf + st[t], tf[t], x);
        mine += all ? 1u : 0u;
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
      count = mine; match = count > 0;
    } else {
      uint32_t res = 0; bool ovf = false;
      if (lane == 0) {
        const uint32_t* L0 = buf; const uint32_t* Ll = buf + st[T - 1];
        if (T == 2) {
          res = P.scoring ? ph_count_slop(L0, tf[0], Ll, tf[1], slop) : (ph_exists_slop(L0, tf[0], Ll, tf[1], slop) ? 1u : 0u);
        } else {
          PhCarry C;
          C.lp = buf + S; C.ls = C.lp + W; C.pb = C.ls + W; C.sb = C.pb + W; C.cap = (uint32_t)W; C.need = 0;
          for (uint32_t i = 0; i < tf[0]; i++) C.lp[i] = L0[i];
          C.llen = tf[0]; C.lslen = 0;
          for (uint32_t t = 1; t + 1 < T && !ovf && C.llen; t++) ph_carry(C, buf + st[t], tf[t], slop, true, &ovf);
          if (!ovf && C.llen) {
            if (P.scoring) res = ph_carry(C, Ll, tf[T - 1], slop, false, &ovf);
            else res = ph_exists_slop(C.lp, C.llen, Ll, tf[T - 1], slop) ? 1u : 0u;
          }
          if (ovf) {   // ov[3] = max(ov[3], merge length asked for / S)
            const unsigned int want = (unsigned int)min((C.need + S - 1) / S, (uint64_t)0xFFFFFFFFu);
            unsigned int* m = (unsigned int*)(P.ov + 3);   // the low word (little endian); the high word stays 0
            unsigned int old = *m;
            while (old < want) { const unsigned int seen = atomicCAS(m, old, want); if (seen == old) break; old = seen; }
          }
        }
      }
      res = __shfl_sync(0xffffffffu, res, 0);
      ovf = __shfl_sync(0xffffffffu, ovf ? 1u : 0u, 0) != 0;
      if (ovf) {   // the carrying merge outgrew its buffers: the next pass has 4x larger ones
        if (lane == 0) { const unsigned long long i = atomicAdd(P.ov + 0, 1ull); P.ov_list[i] = c; atomicAdd(P.ov + 1, (unsigned long long)S); }
        continue;
      }
      count = res; match = res > 0;
    }
    n_dec += S; n_bytes += cand_bytes;
    if (match) {
      if (lane == 0) {
        const uint32_t doc = P.c_doc[e];
        const float score = P.scoring ? a3_term_score(P.q_weight[slot], count, P.cache[P.fieldnorm[doc]]) : 1.0f;
        const uint32_t j = atomicAdd(P.m_cnt + slot, 1u);
        P.m_key[P.cand_off[slot] + j] = ord_f32(score);
        P.m_doc[P.cand_off[slot] + j] = doc;
      }
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

// PositionReader::read for one term (sb200_positions_read): one warp
__global__ void k_positions_read(const PosView V, uint32_t ord, uint64_t offset, uint32_t n, uint32_t* out) {
  __shared__ uint32_t tb[128];
  ph_read_deltas(V, ord, offset, n, out, tb, threadIdx.x & 31);
}

// ------------------------------------------------------------------ directories (attach) ----------------------------------
// one thread per term: [VInt n_blocks] header of the term's positions (reader.rs:43-55)
__global__ void k_pos_header(const uint8_t* __restrict__ file, const uint64_t* __restrict__ poff, const uint64_t* __restrict__ plen,
                             uint32_t n_terms, uint32_t* nblk, uint64_t* hdr, int* err) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_terms) return;
  const uint64_t off = poff[t], end = off + plen[t];
  uint64_t v = 0, p = off; int sh = 0; bool closed = false;
  for (int i = 0; i < 10 && p < end; i++) { const uint8_t b = file[p++]; v |= (uint64_t)(b & 127u) << sh; if (b & 128u) { closed = true; break; } sh += 7; }
  if (!closed || v > 0xFFFFFFFFull || p + v > end) { *err = 1; nblk[t] = 0; hdr[t] = off; return; }
  nblk[t] = (uint32_t)v; hdr[t] = p;
}

// one warp per term: bit widths -> block byte offsets, the tail's extent and value count, and the position offset of every
// posting block from the 12-byte skip entries (tf sum at bytes 6..9, skip.rs:217-232)
__global__ void k_pos_dir(const uint8_t* __restrict__ file, const uint64_t* __restrict__ poff, const uint64_t* __restrict__ plen,
                          const uint64_t* __restrict__ hdr, const uint32_t* __restrict__ nblk, const uint32_t* __restrict__ pfirst,
                          uint32_t n_terms, const uint8_t* __restrict__ postings, const uint64_t* __restrict__ t_data_off,
                          const uint32_t* __restrict__ t_df, const uint32_t* __restrict__ t_first,
                          uint64_t* data_off, uint64_t* tail_off, uint64_t* end_off, uint64_t* count, uint64_t* b_off, uint8_t* b_w,
                          uint64_t* pos_base, int* err) {
  const uint32_t t = (blockIdx.x * (uint32_t)blockDim.x + threadIdx.x) >> 5;
  if (t >= n_terms) return;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t nb = nblk[t], first = pfirst[t];
  const uint64_t h = hdr[t], data = h + nb, end = poff[t] + plen[t];
  uint64_t run = 0;
  bool bad = false;
  for (uint32_t base = 0; base < nb; base += 32) {
    const uint32_t j = base + lane;
    const uint32_t w = j < nb ? file[h + j] : 0u;
    if (w > 32) bad = true;
    const uint32_t size = w * 16u;
    const uint32_t incl = warp_scan_incl(size, lane);
    if (j < nb) { b_off[first + j] = run + incl - size; b_w[first + j] = (uint8_t)w; }
    run += __shfl_sync(0xffffffffu, incl, 31);
  }
  const uint64_t tail = data + run;
  uint32_t stops = 0;
  if (tail > end) bad = true;
  else {
    for (uint64_t base = tail; base < end; base += 32) {
      const uint64_t b = base + lane;
      const bool stop = b < end && (file[b] & 0x80u);
      stops += __popc(__ballot_sync(0xffffffffu, stop));
    }
    if (stops > 127 || (end > tail && !(file[end - 1] & 0x80u))) bad = true;
  }
  if (lane == 0) { data_off[t] = data; tail_off[t] = min(tail, end); end_off[t] = end; count[t] = (uint64_t)nb * 128u + stops; }
  const uint32_t nfull = t_df[t] >> 7, pf = t_first[t];
  const uint8_t* skip = postings + t_data_off[t] - (uint64_t)nfull * 12u;
  unsigned long long acc = 0;
  for (uint32_t base = 0; base < nfull; base += 32) {
    const uint32_t j = base + lane;
    unsigned long long v = 0;
    if (j < nfull) { const uint8_t* s = skip + (uint64_t)j * 12u + 6u; v = (uint32_t)s[0] | ((uint32_t)s[1] << 8) | ((uint32_t)s[2] << 16) | ((uint32_t)s[3] << 24); }
    unsigned long long incl = v;
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long x = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (uint32_t)o) incl += x; }
    if (j < nfull) pos_base[pf + j] = acc + incl - v;
    acc += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (lane == 0) pos_base[pf + nfull] = acc;
  if (__any_sync(0xffffffffu, bad) && lane == 0) *err = 2;
}

}  // namespace sb200
