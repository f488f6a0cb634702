// oracle/oracle_postings.cpp -- CPU restatement of the reference's BM25 posting-list path.
// TEST INFRASTRUCTURE ONLY (see oracle_common.h).  Follows, by file:line in /root/reference/crates:
//   tantivy/src/postings/compression/mod.rs:1-160, vint.rs          block / vint codec
//   tantivy/src/postings/skip.rs:13-281                              skip entries, SkipReader
//   tantivy/src/postings/serializer.rs:294-462                       PostingsSerializer (writer)
//   tantivy/src/postings/block_segment_postings.rs:36-375            BlockSegmentPostings cursor
//   tantivy/src/postings/segment_postings.rs:154-233, block_search.rs:23-34   SegmentPostings
//   tantivy/src/fieldnorm/code.rs                                    fieldnorm <-> id
//   tantivy/src/query/bm25.rs:52-196                                 tantivy Bm25Weight (f32)
//   tantivy/src/query/term_query/term_scorer.rs:9-124                TermScorer
//   tantivy/src/query/intersection.rs:14-160                         Intersection
//   tantivy/src/query/boolean_query/block_wand.rs:16-260             Block-WAND
//   tantivy/src/query/weight.rs:47-60                                for_each_pruning_scorer
//   tantivy/src/collector/top_score_collector.rs:385-564, top_collector.rs:50-66   TopNComputer
//   core/src/ranking/bm25.rs:23-151, computer/mod.rs:61-124, initial.rs:79-93      Stract BM25 + combine
//
// Third-party arithmetic not under /root/reference: `bitpacking` 0.9.2 (BitPacker4x).  Its published
// layout is restated here: 128 ints = 32 rows x 4 lanes, int k in lane k%4 at position k/4, each
// lane an independent little-endian bit stream of num_bits-wide values over 32-bit words, the words
// of the 4 lanes interleaved (u32 index = word*4 + lane); strictly-sorted variant packs
// v[k]-v[k-1]-1 with initial None == u32::MAX (wrapping), i.e. the first value verbatim.
// The reference's tests pin round trips and sizes only, never packed bytes: BYTE-LAYOUT PARITY
// UNPINNED, decoded-value parity pinned (tests/test_oracle_path2.py).
#include "oracle_common.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <thread>
#include <atomic>
#include <vector>

static const uint32_t TERMINATED = 0x7FFFFFFFu;  // tantivy/src/docset.rs:9 (i32::MAX)
static const int BLOCK = 128;

// ---------------------------------------------------------------- fieldnorm code -------------
static uint32_t fieldnorm_table[256];
static struct FieldnormInit {
  FieldnormInit() {  // fieldnorm/code.rs:298-318 (the formula the table is tested against)
    for (int b = 0; b < 256; b++) {
      if (b < 24) { fieldnorm_table[b] = b; continue; }
      uint32_t x = b - 24, bits = x & 7, shift = x >> 3;
      uint32_t v = (shift == 0) ? bits : ((bits | 8u) << (shift - 1));
      fieldnorm_table[b] = 24 + v;
    }
  }
} fieldnorm_init_;
ORC_API uint32_t orc_id_to_fieldnorm(uint8_t id) { return fieldnorm_table[id]; }
ORC_API uint8_t orc_fieldnorm_to_id(uint32_t fn) {  // binary_search(...).unwrap_or_else(|i| i-1)
  const uint32_t* e = std::upper_bound(fieldnorm_table, fieldnorm_table + 256, fn);
  return (uint8_t)((e - fieldnorm_table) - 1);
}

// ---------------------------------------------------------------- BitPacker4x ----------------
static inline uint8_t bit_len(uint32_t v) { return v == 0 ? 0 : (uint8_t)(32 - __builtin_clz(v)); }

static size_t bp4_pack(const uint32_t* vals /*128*/, uint8_t nb, uint8_t* out) {
  if (nb == 0) return 0;
  std::vector<uint32_t> words((size_t)nb * 4, 0u);
  for (int k = 0; k < BLOCK; k++) {
    const int lane = k & 3, pos = k >> 2;
    const uint64_t bit = (uint64_t)pos * nb;
    const int w = (int)(bit >> 5), sh = (int)(bit & 31);
    const uint64_t v = (uint64_t)(nb == 32 ? vals[k] : (vals[k] & ((1u << nb) - 1u))) << sh;
    words[(size_t)w * 4 + lane] |= (uint32_t)v;
    if (sh + nb > 32) words[(size_t)(w + 1) * 4 + lane] |= (uint32_t)(v >> 32);
  }
  memcpy(out, words.data(), (size_t)nb * 16);
  return (size_t)nb * 16;
}
static size_t bp4_unpack(const uint8_t* in, uint8_t nb, uint32_t* vals /*128*/) {
  if (nb == 0) { for (int k = 0; k < BLOCK; k++) vals[k] = 0; return 0; }
  std::vector<uint32_t> words((size_t)nb * 4);
  memcpy(words.data(), in, (size_t)nb * 16);
  const uint64_t mask = (nb == 32) ? 0xFFFFFFFFull : ((1ull << nb) - 1ull);
  for (int k = 0; k < BLOCK; k++) {
    const int lane = k & 3, pos = k >> 2;
    const uint64_t bit = (uint64_t)pos * nb;
    const int w = (int)(bit >> 5), sh = (int)(bit & 31);
    uint64_t x = words[(size_t)w * 4 + lane];
    if (sh + nb > 32) x |= (uint64_t)words[(size_t)(w + 1) * 4 + lane] << 32;
    vals[k] = (uint32_t)((x >> sh) & mask);
  }
  return (size_t)nb * 16;
}
// compress_block_sorted (compression/mod.rs:33-44): offset 0 -> None -> first value verbatim
static size_t block_pack_sorted(const uint32_t* docs, uint32_t offset, uint8_t* nb_out, uint8_t* out) {
  uint32_t d[BLOCK];
  uint32_t prev = (offset == 0) ? 0xFFFFFFFFu : offset;
  uint32_t mx = 0;
  for (int k = 0; k < BLOCK; k++) { d[k] = docs[k] - prev - 1u; prev = docs[k]; mx |= d[k]; }
  *nb_out = bit_len(mx);
  return bp4_pack(d, *nb_out, out);
}
static size_t block_unpack_sorted(const uint8_t* in, uint32_t offset, uint8_t nb, bool strict, uint32_t* docs) {
  uint32_t d[BLOCK];
  size_t used = bp4_unpack(in, nb, d);
  if (strict) {
    uint32_t prev = (offset == 0) ? 0xFFFFFFFFu : offset;
    for (int k = 0; k < BLOCK; k++) { prev = prev + d[k] + 1u; docs[k] = prev; }
  } else {
    uint32_t prev = offset;
    for (int k = 0; k < BLOCK; k++) { prev = prev + d[k]; docs[k] = prev; }
  }
  return used;
}
// compress_block_unsorted(block, minus_one_encoded=true) (compression/mod.rs:52-74)
static size_t block_pack_tf(const uint32_t* tfs, uint8_t* nb_out, uint8_t* out) {
  uint32_t d[BLOCK]; uint32_t mx = 0;
  for (int k = 0; k < BLOCK; k++) { d[k] = tfs[k] - 1u; mx |= d[k]; }
  *nb_out = bit_len(mx);
  return bp4_pack(d, *nb_out, out);
}

// vint (compression/vint.rs): 7-bit groups, little-endian, stop bit 0x80 on the LAST byte
static void vint_put(std::vector<uint8_t>& o, uint32_t v) {
  for (;;) { uint8_t b = v & 127u; v >>= 7; if (v == 0) { o.push_back(b | 128u); break; } o.push_back(b); }
}
static size_t vint_get(const uint8_t* p, uint32_t* v) {
  size_t n = 0; uint32_t r = 0, sh = 0;
  for (;;) { uint8_t b = p[n++]; r += (uint32_t)(b & 127u) << sh; if (b & 128u) break; sh += 7; }
  *v = r; return n;
}

ORC_API uint64_t orc_bp4_roundtrip(const uint32_t* vals, uint8_t nb, uint8_t* packed, uint32_t* back) {
  size_t n = bp4_pack(vals, nb, packed);
  bp4_unpack(packed, nb, back);
  return n;
}
ORC_API uint64_t orc_vint_sorted_encode(const uint32_t* vals, uint32_t n, uint32_t offset, uint8_t* out) {
  std::vector<uint8_t> o;
  for (uint32_t i = 0; i < n; i++) { vint_put(o, vals[i] - offset); offset = vals[i]; }
  memcpy(out, o.data(), o.size());
  return o.size();
}
ORC_API uint8_t orc_encode_bitwidth(uint8_t bw, int delta1) { return bw | ((delta1 ? 1 : 0) << 6); }  // skip.rs:13-15

// ---------------------------------------------------------------- tantivy Bm25Weight ---------
static const float K1 = 1.2f, Bc = 0.75f;
struct TvBm25 {
  float weight; float cache[256];
  static float idf(uint64_t df, uint64_t n) {  // bm25.rs:52-56
    float x = ((float)(n - df) + 0.5f) / ((float)df + 0.5f);
    return logf(1.0f + x);
  }
  void init(float idf_, float avg_fn) {  // bm25.rs:58-68,160-176
    weight = idf_ * (1.0f + K1);
    for (int id = 0; id < 256; id++) cache[id] = K1 * (1.0f - Bc + Bc * (float)fieldnorm_table[id] / avg_fn);
  }
  inline float tf_factor(uint8_t id, uint32_t tf) const { float t = (float)tf; return t / (t + cache[id]); }
  inline float score(uint8_t id, uint32_t tf) const { return weight * tf_factor(id, tf); }
  inline float max_score() const { return score(255, 2013265944u); }
};
ORC_API float orc_tv_idf(uint64_t df, uint64_t n) { return TvBm25::idf(df, n); }
ORC_API void orc_tv_bm25_weight(float idf, float avg_fn, float* weight, float* cache256) {
  TvBm25 w; w.init(idf, avg_fn); *weight = w.weight; memcpy(cache256, w.cache, sizeof(w.cache));
}
ORC_API float orc_tv_bm25_score(float weight, const float* cache256, uint8_t fn_id, uint32_t tf) {
  float t = (float)tf; return weight * (t / (t + cache256[fn_id]));
}
// Stract's own weight (core/src/ranking/bm25.rs:29-45,110-151): weight = idf, (tf*(k1+1))/(tf+cache), tf==0 -> 0
ORC_API void orc_stract_bm25_weight(float idf, float avg_fn, float k1, float b, float* weight, float* cache256) {
  *weight = idf;
  for (int id = 0; id < 256; id++) cache256[id] = k1 * (1.0f - b + b * (float)fieldnorm_table[id] / avg_fn);
}
static inline float stract_score(float weight, const float* cache, float k1, uint8_t id, uint32_t tf) {
  if (tf == 0) return 0.0f;
  float t = (float)tf;
  return weight * ((t * (k1 + 1.0f)) / (t + cache[id]));
}
ORC_API float orc_stract_bm25_score(float weight, const float* cache256, float k1, uint8_t id, uint32_t tf) {
  return stract_score(weight, cache256, k1, id, tf);
}

// ---------------------------------------------------------------- segment (writer side) ------
struct TermInfo { uint64_t off, len; uint32_t df; };
struct Segment {
  std::vector<uint8_t> postings;      // the ".idx" postings file of one field
  std::vector<TermInfo> terms;
  std::vector<uint8_t> fieldnorm_ids; // 1 byte per doc
  uint32_t max_doc = 0;
  float avg_fieldnorm = 0;            // total_num_tokens / max_doc (f32), bm25.rs:112-114
  uint64_t total_tokens = 0;
  int record = 1;                     // IndexRecordOption: 1 WithFreqs (8-byte skip entries), 2 WithFreqsAndPositions (12)
};

ORC_API void* orc_seg_new(const uint8_t* fieldnorm_ids, uint32_t max_doc) {
  Segment* s = new Segment();
  s->fieldnorm_ids.assign(fieldnorm_ids, fieldnorm_ids + max_doc);
  s->max_doc = max_doc;
  uint64_t tot = 0;
  for (uint32_t d = 0; d < max_doc; d++) tot += fieldnorm_table[fieldnorm_ids[d]];
  s->total_tokens = tot;
  s->avg_fieldnorm = max_doc ? (float)tot / (float)max_doc : 0.0f;
  return s;
}
ORC_API void orc_seg_free(void* h) { delete (Segment*)h; }
ORC_API float orc_seg_avg_fieldnorm(void* h) { return ((Segment*)h)->avg_fieldnorm; }
ORC_API void orc_seg_set_avg_fieldnorm(void* h, float a) { ((Segment*)h)->avg_fieldnorm = a; }
ORC_API void orc_seg_set_record(void* h, int record) { ((Segment*)h)->record = record; }

// PostingsSerializer for one term, IndexRecordOption::WithFreqs (serializer.rs:343-462)
ORC_API uint32_t orc_seg_add_term(void* h, const uint32_t* docs, const uint32_t* tfs, uint32_t df) {
  Segment* s = (Segment*)h;
  std::vector<uint8_t> skip, post;
  TvBm25 bw; bool have_bw = s->max_doc != 0;
  if (have_bw) bw.init(TvBm25::idf(df, s->max_doc), s->avg_fieldnorm);  // new_term :343-365
  uint32_t last = 0;
  uint8_t buf[BLOCK * 4];
  uint32_t nfull = df / BLOCK;
  for (uint32_t b = 0; b < nfull; b++) {  // write_block :367-416
    const uint32_t* bd = docs + (size_t)b * BLOCK; const uint32_t* bt = tfs + (size_t)b * BLOCK;
    uint8_t nb; size_t n = block_pack_sorted(bd, last, &nb, buf);
    last = bd[BLOCK - 1];
    for (int i = 0; i < 4; i++) skip.push_back((uint8_t)(last >> (8 * i)));
    skip.push_back(nb | 0x40);  // encode_bitwidth(num_bits, true)
    post.insert(post.end(), buf, buf + n);
    uint8_t tnb; n = block_pack_tf(bt, &tnb, buf);
    post.insert(post.end(), buf, buf + n);
    skip.push_back(tnb);
    if (s->record == 2) {  // write_total_term_freq (skip.rs:65-67), only with positions (serializer.rs:383-388)
      uint32_t sum = 0;
      for (int k = 0; k < BLOCK; k++) sum += bt[k];
      for (int i = 0; i < 4; i++) skip.push_back((uint8_t)(sum >> (8 * i)));
    }
    uint8_t best_id = 0; uint32_t best_tf = 0;
    if (have_bw) {  // max_by keeps the LAST maximum under partial_cmp
      float best = -1.0f; bool first = true;
      for (int k = 0; k < BLOCK; k++) {
        uint8_t id = s->fieldnorm_ids[bd[k]];
        float f = bw.tf_factor(id, bt[k]);
        if (first || !(f < best)) { best = f; best_id = id; best_tf = bt[k]; first = false; }
      }
    }
    skip.push_back(best_id);
    skip.push_back((uint8_t)std::min<uint32_t>(best_tf, 255u));
  }
  const uint32_t rem = df - nfull * BLOCK;  // close_term :428-462
  if (rem) {
    uint32_t off = last;
    for (uint32_t i = 0; i < rem; i++) { uint32_t v = docs[(size_t)nfull * BLOCK + i]; vint_put(post, v - off); off = v; }
    for (uint32_t i = 0; i < rem; i++) vint_put(post, tfs[(size_t)nfull * BLOCK + i]);
  }
  TermInfo ti; ti.off = s->postings.size(); ti.df = df;
  if (df >= (uint32_t)BLOCK) {
    uint64_t v = skip.size();  // common VInt: same 7-bit / stop-bit-last convention
    for (;;) { uint8_t bte = v & 127u; v >>= 7; if (v == 0) { s->postings.push_back(bte | 128u); break; } s->postings.push_back(bte); }
    s->postings.insert(s->postings.end(), skip.begin(), skip.end());
  }
  s->postings.insert(s->postings.end(), post.begin(), post.end());
  ti.len = s->postings.size() - ti.off;
  s->terms.push_back(ti);
  return (uint32_t)s->terms.size() - 1;
}
ORC_API uint64_t orc_seg_postings_len(void* h) { return ((Segment*)h)->postings.size(); }
ORC_API void orc_seg_postings_copy(void* h, uint8_t* out) { Segment* s = (Segment*)h; memcpy(out, s->postings.data(), s->postings.size()); }
ORC_API uint32_t orc_seg_num_terms(void* h) { return (uint32_t)((Segment*)h)->terms.size(); }
ORC_API void orc_seg_term_info(void* h, uint32_t t, uint64_t* off, uint64_t* len, uint32_t* df) {
  const TermInfo& ti = ((Segment*)h)->terms[t]; *off = ti.off; *len = ti.len; *df = ti.df;
}
// adopt externally produced bytes (used to check that the library and the oracle parse the same file)
ORC_API void orc_seg_set_postings(void* h, const uint8_t* bytes, uint64_t len, const uint64_t* offs, const uint64_t* lens,
                                  const uint32_t* dfs, uint32_t n_terms) {
  Segment* s = (Segment*)h;
  s->postings.assign(bytes, bytes + len);
  s->terms.resize(n_terms);
  for (uint32_t i = 0; i < n_terms; i++) s->terms[i] = {offs[i], lens[i], dfs[i]};
}

// ---------------------------------------------------------------- cursors --------------------
struct SkipReader {  // skip.rs:85-281: WithFreqs (8-byte entries) and WithFreqsAndPositions (12-byte entries)
  const uint8_t* p = nullptr;
  int record = 1;
  uint32_t last_doc_in_block = 0, last_doc_in_previous_block = 0, remaining = 0;
  size_t byte_offset = 0;
  bool bitpacked = false; uint8_t doc_bits = 0, tf_bits = 0, bw_id = 0; bool strict = true; uint32_t bw_tf = 0, vint_docs = 0;
  void read_block_info() {
    last_doc_in_block = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
    doc_bits = p[4] & 0x3f; strict = (p[4] >> 6) & 1;
    tf_bits = p[5];
    const int bw = record == 2 ? 10 : 6;  // skip.rs:203-232: tf_sum u32 sits before the block-wand pair
    bw_id = p[bw]; bw_tf = (p[bw + 1] == 255) ? 0xFFFFFFFFu : p[bw + 1];
    bitpacked = true; p += (record == 2 ? 12 : 8);
  }
  void reset(const uint8_t* data, uint32_t df, int rec) {
    record = rec;
    last_doc_in_block = df >= (uint32_t)BLOCK ? 0 : TERMINATED;
    last_doc_in_previous_block = 0; p = data; bitpacked = false; vint_docs = df; byte_offset = 0; remaining = df;
    if (df >= (uint32_t)BLOCK) read_block_info();
  }
  void advance() {
    if (bitpacked) { remaining -= BLOCK; byte_offset += (size_t)(doc_bits + tf_bits) * 16; }
    else { remaining = 0; byte_offset = (size_t)-1; }
    last_doc_in_previous_block = last_doc_in_block;
    if (remaining >= (uint32_t)BLOCK) read_block_info();
    else { last_doc_in_block = TERMINATED; bitpacked = false; vint_docs = remaining; }
  }
  bool seek(uint32_t target) {
    if (last_doc_in_block >= target) return false;
    for (;;) { advance(); if (last_doc_in_block >= target) return true; }
  }
};

struct Postings {  // BlockSegmentPostings + SegmentPostings
  const Segment* seg = nullptr;
  const uint8_t* data = nullptr;  // posting bytes after the skip section
  uint32_t df = 0;
  SkipReader skip;
  uint32_t docs[BLOCK], tfs[BLOCK];
  uint32_t block_len = 0; bool loaded = false;
  bool has_bm_cache = false; float bm_cache = 0;
  uint32_t cur = 0;
  void open(const Segment* s, uint32_t term) {
    seg = s; const TermInfo& ti = s->terms[term]; df = ti.df;
    const uint8_t* b = s->postings.data() + ti.off;
    const uint8_t* skipdata = nullptr;
    if (df >= (uint32_t)BLOCK) {  // split_into_skips_and_postings :78-88
      uint64_t sl = 0; int sh = 0;
      for (;;) { uint8_t x = *b++; sl |= (uint64_t)(x & 127u) << sh; if (x & 128u) break; sh += 7; }
      skipdata = b; b += sl;
    }
    data = b;
    skip.reset(skipdata, df, s->record);
    loaded = false; has_bm_cache = false; cur = 0;
    load_block();
  }
  void load_block() {  // :303-351
    if (loaded) return;
    if (skip.bitpacked) {
      const uint8_t* d = data + skip.byte_offset;
      size_t used = block_unpack_sorted(d, skip.last_doc_in_previous_block, skip.doc_bits, skip.strict, docs);
      uint32_t t[BLOCK]; bp4_unpack(d + used, skip.tf_bits, t);
      for (int k = 0; k < BLOCK; k++) tfs[k] = t[k] + (skip.strict ? 1u : 0u);
      block_len = BLOCK;
    } else {
      for (int k = 0; k < BLOCK; k++) { docs[k] = TERMINATED; tfs[k] = TERMINATED; }
      uint32_t n = skip.vint_docs;
      if (n) {
        const uint8_t* d = data + skip.byte_offset;
        uint32_t off = skip.last_doc_in_previous_block;
        for (uint32_t i = 0; i < n; i++) { uint32_t v; d += vint_get(d, &v); off += v; docs[i] = off; }
        for (uint32_t i = 0; i < n; i++) { uint32_t v; d += vint_get(d, &v); tfs[i] = v; }
      }
      block_len = n;
    }
    loaded = true;
  }
  void shallow_seek(uint32_t target) { if (skip.seek(target)) { has_bm_cache = false; loaded = false; } }
  void block_seek(uint32_t target) { shallow_seek(target); load_block(); }
  void block_advance() { skip.advance(); loaded = false; has_bm_cache = false; load_block(); }
  // DocSet
  inline uint32_t doc() const { return docs[cur]; }
  inline uint32_t term_freq() const { return tfs[cur]; }
  uint32_t advance() {  // segment_postings.rs:157-166
    if (cur == BLOCK - 1) { cur = 0; block_advance(); } else cur++;
    return doc();
  }
  uint32_t seek(uint32_t target) {  // :168-193 + branchless_binary_search
    if (doc() >= target) return doc();
    block_seek(target);
    uint32_t start = 0, len = BLOCK;
    for (int i = 0; i < 7; i++) { len /= 2; if (docs[start + len - 1] < target) start += len; }
    cur = start;
    return docs[cur];
  }
  float block_max_score(const TvBm25& w) {  // block_segment_postings.rs:147-184
    if (has_bm_cache) return bm_cache;
    if (skip.bitpacked) { bm_cache = w.score(skip.bw_id, skip.bw_tf); has_bm_cache = true; return bm_cache; }
    if (loaded) {
      float best = 0.0f; bool first = true;
      for (uint32_t i = 0; i < block_len; i++) {
        float sc = w.score(seg->fieldnorm_ids[docs[i]], tfs[i]);
        if (first) { best = sc; first = false; } else best = std::fmax(best, sc);
      }
      bm_cache = first ? 0.0f : best; has_bm_cache = true; return bm_cache;
    }
    return w.max_score();
  }
};

struct TermScorer {  // term_scorer.rs
  Postings post; TvBm25 w; const Segment* seg; float max_sc; uint32_t ord;
  inline uint32_t doc() const { return post.doc(); }
  inline float score() const { return w.score(seg->fieldnorm_ids[post.doc()], post.term_freq()); }
  inline uint32_t advance() { return post.advance(); }
  inline uint32_t seek(uint32_t t) { return post.seek(t); }
  inline uint32_t last_doc_in_block() const { return post.skip.last_doc_in_block; }
  inline void shallow_seek(uint32_t t) { post.shallow_seek(t); }
  inline float block_max_score() { return post.block_max_score(w); }
};

// ---------------------------------------------------------------- TopNComputer ---------------
// Order keys.  f32 BM25 scores are finite and >= 0: plain `>`.  f64 recall totals may be negative, -0.0, +-inf or NaN:
// f64::total_cmp over the bits (the reference's ScoredDoc::cmp, collector/top_docs.rs:229-233), -0.0 below +0.0, with every
// NaN first made the one negative quiet NaN 0xFFF8000000000000, so all NaN totals tie below -inf whatever sign their
// computation left (DESIGN §5).  The device's ord_f64 (bm25.cu) is the same map.
static inline float order_key(float f) { return f; }
static inline uint64_t order_key(double f) {
  uint64_t b; memcpy(&b, &f, 8);
  if (f != f) b = 0xFFF8000000000000ull;
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
template <class S>
struct TopN {  // top_score_collector.rs:440-564 with ComparableDoc order (score desc, doc asc)
  struct E { S feature; uint32_t doc; };
  std::vector<E> buf; size_t top_n, cap; bool has_thr = false; S thr{};
  explicit TopN(size_t n) : top_n(n), cap(std::max<size_t>(n, 1) * 2) { buf.reserve(cap); }
  static bool before(const E& a, const E& b) {
    const auto ka = order_key(a.feature), kb = order_key(b.feature);
    if (ka != kb) return ka > kb;
    return a.doc < b.doc;
  }
  S truncate() {
    std::nth_element(buf.begin(), buf.begin() + top_n, buf.end(), before);
    S med = buf[top_n].feature;
    buf.resize(top_n);
    return med;
  }
  void push(S f, uint32_t d) {
    if (has_thr && order_key(f) < order_key(thr)) return;
    if (buf.size() == cap) { thr = truncate(); has_thr = true; }
    buf.push_back({f, d});
  }
  std::vector<E> into_sorted() {
    if (buf.size() > top_n) truncate();
    std::sort(buf.begin(), buf.end(), before);
    return buf;
  }
};

struct QueryTerm { uint32_t term; float weight; const float* cache; };

static void make_scorers(const Segment* s, const uint32_t* terms, const float* weights, const float* caches, uint32_t n,
                         std::vector<TermScorer>& out) {
  out.resize(n);
  for (uint32_t i = 0; i < n; i++) {
    out[i].seg = s; out[i].ord = i;
    out[i].w.weight = weights[i]; memcpy(out[i].w.cache, caches + (size_t)i * 256, 256 * sizeof(float));
    out[i].max_sc = out[i].w.max_score();
    out[i].post.open(s, terms[i]);
  }
}

// BooleanQuery of Must TermQueries + TopDocs::with_limit(k): intersect_scorers + for_each_pruning_scorer
static uint32_t and_topk(const Segment* s, const uint32_t* terms, const float* weights, const float* caches, uint32_t n,
                         uint32_t k, uint32_t* out_docs, float* out_scores, uint64_t* scored) {
  std::vector<TermScorer> sc;
  make_scorers(s, terms, weights, caches, n, sc);
  TopN<float> top(k);
  float threshold = -3.4028235e38f;  // Score::MIN
  uint64_t nscored = 0;
  auto emit = [&](uint32_t doc, float score) {
    nscored++;
    if (score > threshold) { top.push(score, doc); threshold = top.has_thr ? top.thr : -3.4028235e38f; }
  };
  if (n == 1) {  // BooleanWeight with one clause defers to the TermWeight: block_wand_single_scorer (term_weight.rs:81-90)
    TermScorer& t = sc[0];
    uint32_t doc = t.doc();
    for (;;) {
      bool done = false;
      while (t.block_max_score() < threshold) {
        uint32_t l = t.last_doc_in_block();
        if (l == TERMINATED) { done = true; break; }
        doc = l + 1; t.shallow_seek(doc);
      }
      if (done) break;
      doc = t.seek(doc);
      if (doc == TERMINATED) break;
      bool ret = false;
      for (;;) {
        emit(doc, t.score());
        if (doc == t.last_doc_in_block()) break;
        doc = t.advance();
        if (doc == TERMINATED) { ret = true; break; }
      }
      if (ret) break;
      doc += 1; t.shallow_seek(doc);
    }
  } else {
    std::vector<TermScorer*> o(n);
    for (uint32_t i = 0; i < n; i++) o[i] = &sc[i];
    std::stable_sort(o.begin(), o.end(), [](TermScorer* a, TermScorer* b) { return a->post.df < b->post.df; });  // sort_by_key(size_hint)
    // go_to_first_doc (intersection.rs:53-66)
    uint32_t cand = 0;
    for (auto* t : o) cand = std::max(cand, t->doc());
    for (bool again = true; again;) {
      again = false;
      for (auto* t : o) { uint32_t sd = t->seek(cand); if (sd > cand) { cand = t->doc(); again = true; break; } }
    }
    uint32_t doc = cand;
    TermScorer *left = o[0], *right = o[1];
    while (doc != TERMINATED) {
      float others = 0.0f;
      for (uint32_t i = 2; i < n; i++) others += o[i]->score();
      emit(doc, left->score() + right->score() + others);
      // Intersection::advance (intersection.rs:96-125)
      uint32_t c = left->advance();
      for (;;) {
        for (;;) { uint32_t rd = right->seek(c); c = left->seek(rd); if (c == rd) break; }
        bool restart = false;
        for (uint32_t i = 2; i < n; i++) { uint32_t sd = o[i]->seek(c); if (sd > c) { c = left->seek(sd); restart = true; break; } }
        if (!restart) break;
      }
      doc = c;
    }
  }
  auto v = top.into_sorted();
  for (size_t i = 0; i < v.size(); i++) { out_docs[i] = v[i].doc; out_scores[i] = v[i].feature; }
  if (scored) *scored = nscored;
  return (uint32_t)v.size();
}

// Should-only TermQueries with freqs: block_wand (block_wand.rs:148-214)
static uint32_t or_topk(const Segment* s, const uint32_t* terms, const float* weights, const float* caches, uint32_t n,
                        uint32_t k, uint32_t* out_docs, float* out_scores, uint64_t* scored) {
  std::vector<TermScorer> store;
  make_scorers(s, terms, weights, caches, n, store);
  if (n == 1) return and_topk(s, terms, weights, caches, n, k, out_docs, out_scores, scored);
  TopN<float> top(k);
  float threshold = -3.4028235e38f;
  uint64_t nscored = 0;
  std::vector<TermScorer*> sc;
  for (auto& t : store) sc.push_back(&t);
  auto by_doc = [](TermScorer* a, TermScorer* b) { return a->doc() < b->doc(); };
  std::stable_sort(sc.begin(), sc.end(), by_doc);
  auto restore = [&](size_t ord) {
    uint32_t d = sc[ord]->doc();
    for (size_t i = ord + 1; i < sc.size(); i++) { if (sc[i]->doc() >= d) break; std::swap(sc[i], sc[i - 1]); }
  };
  for (;;) {
    // find_pivot_doc
    float ms = 0.0f; size_t before = 0; uint32_t pivot = TERMINATED;
    while (before < sc.size()) { ms += sc[before]->max_sc; if (ms > threshold) { pivot = sc[before]->doc(); break; } before++; }
    if (pivot == TERMINATED) break;
    size_t plen = before + 1;
    while (plen < sc.size() && sc[plen]->doc() == pivot) plen++;
    float ub = 0.0f;
    for (size_t i = 0; i < plen; i++) { sc[i]->shallow_seek(pivot); ub += sc[i]->block_max_score(); }
    if (ub <= threshold) {  // block_max_was_too_low_advance_one_scorer
      size_t to_seek = plen - 1; float gmax = sc[to_seek]->max_sc; uint32_t after = sc[to_seek]->last_doc_in_block();
      for (size_t i = plen - 1; i-- > 0;) {
        if (sc[i]->last_doc_in_block() <= after) after = sc[i]->last_doc_in_block();
        if (sc[i]->max_sc > gmax) { gmax = sc[i]->max_sc; to_seek = i; }
      }
      if (after != TERMINATED) after += 1;
      for (size_t i = plen; i < sc.size(); i++) if (sc[i]->doc() <= after) after = sc[i]->doc();
      sc[to_seek]->seek(after);
      restore(to_seek);
      continue;
    }
    // align_scorers
    bool aligned = true;
    for (size_t i = before; i-- > 0;) {
      uint32_t nd = sc[i]->seek(pivot);
      if (nd != pivot) {
        if (nd == TERMINATED) { sc[i] = sc.back(); sc.pop_back(); }  // swap_remove
        if (i < sc.size()) restore(i);
        aligned = false; break;
      }
    }
    if (!aligned) continue;
    float score = 0.0f;
    for (size_t i = 0; i < plen; i++) score += sc[i]->score();
    nscored++;
    if (score > threshold) { top.push(score, pivot); threshold = top.has_thr ? top.thr : -3.4028235e38f; }
    // advance_all_scorers_on_pivot
    for (size_t i = 0; i < plen; i++) sc[i]->advance();
    for (size_t i = 0; i != sc.size();) { if (sc[i]->doc() == TERMINATED) { sc[i] = sc.back(); sc.pop_back(); } else i++; }
    std::stable_sort(sc.begin(), sc.end(), by_doc);
  }
  auto v = top.into_sorted();
  for (size_t i = 0; i < v.size(); i++) { out_docs[i] = v[i].doc; out_scores[i] = v[i].feature; }
  if (scored) *scored = nscored;
  return (uint32_t)v.size();
}

// exhaustive union with query-order f32 sums: what a non-pruning `for_each` over Union<SumCombiner> built from
// scorers that never reorder would give.  Used to (a) cross-check block_wand as the reference's proptests do
// (block_wand.rs:336-508) and (b) define the library's canonical OR order for >= 3 terms.
static uint32_t or_topk_exhaustive(const Segment* s, const uint32_t* terms, const float* weights, const float* caches,
                                   uint32_t n, uint32_t k, uint32_t* out_docs, float* out_scores, uint64_t* scored) {
  std::vector<TermScorer> sc;
  make_scorers(s, terms, weights, caches, n, sc);
  TopN<float> top(k);
  uint64_t nscored = 0;
  for (;;) {
    uint32_t d = TERMINATED;
    for (auto& t : sc) d = std::min(d, t.doc());
    if (d == TERMINATED) break;
    float score = 0.0f;
    for (auto& t : sc) if (t.doc() == d) { score += t.score(); t.advance(); }
    nscored++;
    top.push(score, d);
  }
  auto v = top.into_sorted();
  for (size_t i = 0; i < v.size(); i++) { out_docs[i] = v[i].doc; out_scores[i] = v[i].feature; }
  if (scored) *scored = nscored;
  return (uint32_t)v.size();
}

ORC_API uint32_t orc_bm25_topk(void* seg, const uint32_t* terms, const float* weights, const float* caches, uint32_t n_terms,
                               int mode /*0 AND, 1 OR block-wand, 2 OR exhaustive*/, uint32_t k, uint32_t* docs, float* scores,
                               uint64_t* scored) {
  const Segment* s = (const Segment*)seg;
  if (n_terms == 0 || k == 0) return 0;
  if (mode == 0) return and_topk(s, terms, weights, caches, n_terms, k, docs, scores, scored);
  if (mode == 1) return or_topk(s, terms, weights, caches, n_terms, k, docs, scores, scored);
  return or_topk_exhaustive(s, terms, weights, caches, n_terms, k, docs, scores, scored);
}

// TopN<double> over a caller's (total, doc) list in the given push order, for hand-made lists of special values
ORC_API uint32_t orc_topn_f64(const double* totals, const uint32_t* docs, uint32_t n, uint32_t k, uint32_t* out_docs, double* out_totals) {
  if (k == 0) return 0;
  TopN<double> top(k);
  for (uint32_t i = 0; i < n; i++) top.push(totals[i], docs[i]);
  auto v = top.into_sorted();
  for (size_t i = 0; i < v.size(); i++) { out_docs[i] = v[i].doc; out_totals[i] = v[i].feature; }
  return (uint32_t)v.size();
}

// Stract recall stage on one text field (path 2B): MainCollector over the Should-union of the query terms
// (requires_scoring()==false -> for_each_no_score, ascending docs), per doc
//   total = coeff_text * (bm25 as f64) + sum_j coeff_j * signal_j[doc]          (initial.rs:79-93, order.rs:63-84)
// with bm25 = f32 sum over the query terms in query order of Stract's Bm25Weight::score, tf = 0 when the
// term's posting does not contain the doc (computer/mod.rs:109-124, bm25.rs:97-102,136-150); top-k by
// (total desc, doc asc).  max_docs > 0 mirrors ShortCircuitQuery (stop after that many candidate docs).
ORC_API uint32_t orc_signal_topk(void* seg, const uint32_t* terms, const float* weights, const float* caches, float k1,
                                 uint32_t n_terms, double coeff_text, const double* const* signals, const double* coeffs,
                                 uint32_t n_signals, uint32_t max_docs, uint32_t k, uint32_t* docs, double* totals,
                                 uint64_t* scored) {
  const Segment* s = (const Segment*)seg;
  if (n_terms == 0 || k == 0) return 0;
  std::vector<Postings> cand(n_terms), scorepost(n_terms);
  for (uint32_t i = 0; i < n_terms; i++) { cand[i].open(s, terms[i]); scorepost[i].open(s, terms[i]); }
  TopN<double> top(k);
  uint64_t nscored = 0;
  for (;;) {
    uint32_t d = TERMINATED;
    for (auto& c : cand) d = std::min(d, c.doc());
    if (d == TERMINATED) break;
    for (auto& c : cand) if (c.doc() == d) c.advance();
    const uint8_t id = s->fieldnorm_ids[d];
    float bm = 0.0f;
    for (uint32_t i = 0; i < n_terms; i++) {
      Postings& p = scorepost[i];  // posting_contains: doc()==d || (doc()<d && seek(d)==d)
      uint32_t tf = 0;
      if (p.doc() == d || (p.doc() < d && p.seek(d) == d)) tf = p.term_freq();
      bm += stract_score(weights[i], caches + (size_t)i * 256, k1, id, tf);
    }
    double total = 0.0;
    total += coeff_text * (double)bm;
    for (uint32_t j = 0; j < n_signals; j++) total += coeffs[j] * signals[j][d];
    nscored++;
    top.push(total, d);
    if (max_docs && nscored >= max_docs) break;
  }
  auto v = top.into_sorted();
  for (size_t i = 0; i < v.size(); i++) { docs[i] = v[i].doc; totals[i] = v[i].feature; }
  if (scored) *scored = nscored;
  return (uint32_t)v.size();
}

// Stract recall stage over SEVERAL text fields (SURVEY 8(f) rank 3, first slice): what InitialSegmentScoreTweaker::score
// (initial.rs:79-93) computes from SignalComputeOrder::compute (computer/order.rs:17-135) with the TextFieldData methods of
// computer/mod.rs:66-163.  A field f holds its query terms as "slots" in query order (a term the segment does not know is
// SegmentPostings::empty(): it still counts in num_query_terms and keeps its weights); every method re-seeks the field's
// own cursors (posting_contains, mod.rs:61-63).
//   bm25(f)      f32 sum over the slots of idf * ((tf*(k1+1)) / (tf + cache[fieldnorm_id])), tf = 0 -> 0        (bm25.rs:97-150)
//   bm25f(f)     the same with idf_f (AllBody doc_freq, bm25f.rs:40-45) and tf scaled by the field's signal coefficient
//                as f32 before the saturation (bm25f.rs:167-180)
//   coverage(f)  (number of slots containing the doc as f64) / num_query_terms                                  (mod.rs:91-107)
//   idf_sum(f)   f32 sum of idf over the slots containing the doc                                               (mod.rs:126-143)
// ops are evaluated in the order given (the host mirror derives it like SignalComputeOrder::new): kind 0 bm25(field),
// 1 Bm25F = f64 sum over the fields of bm25f, 2 coverage(field), 3 idf_sum(field), 4 numeric column.  chain != 0 marks an
// n-gram group (largest n first): chain == 1 starts it; score *= 0.4^hits, hits += score > 0 (order.rs:95-135).
// total = f64 sum of coefficient * score in op order.  Candidates = union of all slots' postings, ascending docs.
ORC_API uint32_t orc_multi_signal_topk(uint32_t n_fields, void* const* segs, const float* const* caches, const float* k1s,
                                       const float* coefs, uint32_t n_slots, const uint8_t* slot_field, const uint32_t* slot_term,
                                       const float* slot_idf, const float* slot_idf_f, const double* slot_boost, uint32_t n_ops,
                                       const uint32_t* op_kind,
                                       const uint32_t* op_field, const uint32_t* op_chain, const uint32_t* op_col,
                                       const double* op_coeff, const double* const* signals, uint32_t k, uint32_t* docs,
                                       double* totals, uint64_t* scored) {
  if (k == 0) return 0;
  struct Field { const Segment* seg; std::vector<Postings> post; std::vector<float> idf, idf_f; const float* cache; float k1, coef; };
  std::vector<Field> F(n_fields);
  struct Rule { Postings docset; double boost; };   // RuleBoost (computer/mod.rs:165-172): one posting list per rule here
  std::vector<Rule> rules;
  std::vector<Postings> cand;
  cand.reserve(n_slots);
  for (uint32_t f = 0; f < n_fields; f++) { F[f].seg = (const Segment*)segs[f]; F[f].cache = caches[f]; F[f].k1 = k1s[f]; F[f].coef = coefs[f]; }
  auto open = [](Postings& p, const Segment* s, uint32_t term) {
    if (term == 0xFFFFFFFFu || term >= s->terms.size()) {   // SegmentPostings::empty()
      p.seg = s; p.df = 0; p.skip.reset(nullptr, 0, s->record);
      for (int q = 0; q < BLOCK; q++) { p.docs[q] = TERMINATED; p.tfs[q] = 0; }
      p.block_len = 0; p.loaded = true; p.cur = 0;
    } else p.open(s, term);
  };
  for (uint32_t x = 0; x < n_slots; x++) {
    if (slot_field[x] & 0x80) {   // an optic rule's docset: probed per scored doc, never a source of candidates
      rules.emplace_back(); open(rules.back().docset, F[slot_field[x] & 0x7F].seg, slot_term[x]); rules.back().boost = slot_boost[x];
      continue;
    }
    Field& fd = F[slot_field[x]];
    fd.post.emplace_back(); open(fd.post.back(), fd.seg, slot_term[x]);
    fd.idf.push_back(slot_idf[x]); fd.idf_f.push_back(slot_idf_f[x]);
    cand.emplace_back(); open(cand.back(), fd.seg, slot_term[x]);
  }
  auto contains = [](Postings& p, uint32_t d) { return p.doc() == d || (p.doc() < d && p.seek(d) == d); };
  const double DAMP[3] = {1.0, 0.4, 0.4 * 0.4};   // NGRAM_DAMPENING.powi(hits), hits <= 2 (three n-gram sizes per field)
  TopN<double> top(k);
  uint64_t nscored = 0;
  for (;;) {
    uint32_t d = TERMINATED;
    for (auto& c : cand) d = std::min(d, c.doc());
    if (d == TERMINATED) break;
    for (auto& c : cand) if (c.doc() == d) c.advance();
    double total = 0.0;
    int hits = 0;
    for (uint32_t o = 0; o < n_ops; o++) {
      double sc = 0.0;
      const uint32_t kind = op_kind[o];
      if (kind == 4) sc = signals[op_col[o]][d];
      else if (kind == 1) {
        for (auto& fd : F) {                      // text_fields.values_mut().map(bm25f).sum::<f64>()
          if (fd.post.empty()) continue;          // a field without query terms is not in the map
          const uint8_t id = fd.seg->fieldnorm_ids[d];
          float b = 0.0f;
          for (size_t i = 0; i < fd.post.size(); i++) {
            const uint32_t tf = contains(fd.post[i], d) ? fd.post[i].term_freq() : 0u;
            float part = 0.0f;
            if (tf != 0) { const float t = (float)tf * fd.coef; part = fd.idf_f[i] * ((t * (fd.k1 + 1.0f)) / (t + fd.cache[id])); }
            b += part;
          }
          sc += (double)b;
        }
      } else {
        Field& fd = F[op_field[o]];
        if (!fd.post.empty()) {
          if (kind == 0) {
            const uint8_t id = fd.seg->fieldnorm_ids[d];
            float b = 0.0f;
            for (size_t i = 0; i < fd.post.size(); i++) {
              const uint32_t tf = contains(fd.post[i], d) ? fd.post[i].term_freq() : 0u;
              b += stract_score(fd.idf[i], fd.cache, fd.k1, id, tf);
            }
            sc = (double)b;
          } else if (kind == 2) {
            double n = 0.0;
            for (auto& p : fd.post) n += contains(p, d) ? 1.0 : 0.0;
            sc = n / (double)fd.post.size();
          } else if (kind == 3) {
            float b = 0.0f;
            for (size_t i = 0; i < fd.post.size(); i++) if (contains(fd.post[i], d)) b += fd.idf[i];
            sc = (double)b;
          }
        }
      }
      if (op_chain[o]) {
        if (op_chain[o] == 1) hits = 0;
        sc *= DAMP[hits > 2 ? 2 : hits];
        if (sc > 0.0) hits++;
      }
      total += op_coeff[o] * sc;
    }
    if (slot_boost) {   // SignalComputer::boosts, computer/mod.rs:471-497 (always Some once a segment is registered)
      double downrank = 0.0, boost = 0.0;
      for (auto& r : rules) {
        if (r.docset.doc() > d) continue;
        if (r.docset.doc() == d || r.docset.seek(d) == d) {
          if (r.boost < 0.0) downrank += std::fabs(r.boost); else boost += r.boost;
        }
      }
      total *= (downrank > boost) ? 1.0 / (1.0 + (downrank - boost)) : boost - downrank + 1.0;
    }
    nscored++;
    top.push(total, d);
  }
  auto v = top.into_sorted();
  for (size_t i = 0; i < v.size(); i++) { docs[i] = v[i].doc; totals[i] = v[i].feature; }
  if (scored) *scored = nscored;
  return (uint32_t)v.size();
}

// batch drivers: one query per thread across all host threads (the reference runs a query on one
// thread, tantivy/src/index/index.rs:416, and many queries concurrently)
ORC_API void orc_bm25_topk_batch(void* seg, const uint32_t* terms /*n_q*n_terms*/, const float* weights, const float* caches,
                                 uint32_t n_terms, int mode, uint32_t k, uint32_t n_queries, int threads, uint32_t* docs,
                                 float* scores, uint32_t* n_out, uint64_t* scored) {
  std::atomic<uint32_t> next(0);
  auto work = [&]() {
    for (;;) {
      uint32_t q = next.fetch_add(1);
      if (q >= n_queries) break;
      uint64_t sc = 0;
      n_out[q] = orc_bm25_topk(seg, terms + (size_t)q * n_terms, weights + (size_t)q * n_terms,
                               caches + (size_t)q * n_terms * 256, n_terms, mode, k, docs + (size_t)q * k,
                               scores + (size_t)q * k, &sc);
      if (scored) scored[q] = sc;
    }
  };
  std::vector<std::thread> pool;
  for (int t = 0; t < std::max(threads, 1); t++) pool.emplace_back(work);
  for (auto& th : pool) th.join();
}
ORC_API void orc_signal_topk_batch(void* seg, const uint32_t* terms, const float* weights, const float* caches, float k1,
                                   uint32_t n_terms, double coeff_text, const double* const* signals, const double* coeffs,
                                   uint32_t n_signals, uint32_t max_docs, uint32_t k, uint32_t n_queries, int threads,
                                   uint32_t* docs, double* totals, uint32_t* n_out, uint64_t* scored) {
  std::atomic<uint32_t> next(0);
  auto work = [&]() {
    for (;;) {
      uint32_t q = next.fetch_add(1);
      if (q >= n_queries) break;
      uint64_t sc = 0;
      n_out[q] = orc_signal_topk(seg, terms + (size_t)q * n_terms, weights + (size_t)q * n_terms,
                                 caches + (size_t)q * n_terms * 256, k1, n_terms, coeff_text, signals, coeffs, n_signals,
                                 max_docs, k, docs + (size_t)q * k, totals + (size_t)q * k, &sc);
      if (scored) scored[q] = sc;
    }
  };
  std::vector<std::thread> pool;
  for (int t = 0; t < std::max(threads, 1); t++) pool.emplace_back(work);
  for (auto& th : pool) th.join();
}

// cursor-level hooks for the KATs (term_scorer.rs:142-253)
ORC_API void* orc_cursor_open(void* seg, uint32_t term, float weight, const float* cache256) {
  TermScorer* t = new TermScorer();
  t->seg = (const Segment*)seg; t->w.weight = weight; memcpy(t->w.cache, cache256, sizeof(t->w.cache));
  t->max_sc = t->w.max_score(); t->post.open(t->seg, term);
  return t;
}
ORC_API void orc_cursor_free(void* c) { delete (TermScorer*)c; }
ORC_API uint32_t orc_cursor_doc(void* c) { return ((TermScorer*)c)->doc(); }
ORC_API uint32_t orc_cursor_tf(void* c) { return ((TermScorer*)c)->post.term_freq(); }
ORC_API uint32_t orc_cursor_advance(void* c) { return ((TermScorer*)c)->advance(); }
ORC_API uint32_t orc_cursor_seek(void* c, uint32_t t) { return ((TermScorer*)c)->seek(t); }
ORC_API void orc_cursor_shallow_seek(void* c, uint32_t t) { ((TermScorer*)c)->shallow_seek(t); }
ORC_API float orc_cursor_score(void* c) { return ((TermScorer*)c)->score(); }
ORC_API float orc_cursor_max_score(void* c) { return ((TermScorer*)c)->max_sc; }
ORC_API float orc_cursor_block_max_score(void* c) { return ((TermScorer*)c)->block_max_score(); }
ORC_API uint32_t orc_cursor_last_doc_in_block(void* c) { return ((TermScorer*)c)->last_doc_in_block(); }
ORC_API int orc_p2_proto_marker(void) { return 1; }

// ---------------------------------------------------------------- term info store --------------
// TermInfoStore (tantivy/src/termdict/fst_termdict/term_info_store.rs): blocks of 256 TermInfos; the first of a block
// is stored verbatim in a 47-byte TermInfoBlockMeta (:14-48), the other 255 as bit-packed offsets relative to it
// (:176-262), read back with unaligned 8-byte loads (:102-122,134-153).  BitPacker = tantivy's own LSB-first 64-bit
// mini-buffer (tantivy/src/bitpacker/bitpacker.rs:18-68), compute_num_bits (bitpacker/mod.rs:32-39).
namespace tis {
struct Info { uint32_t df; uint64_t ps, pe, qs, qe; };  // doc_freq, postings range, positions range
struct Packer {
  uint64_t mini = 0; size_t written = 0;
  void write(uint64_t v, uint8_t nb, std::vector<uint8_t>& out) {
    if (written + nb > 64) {
      mini |= (written < 64) ? (v << written) : 0;
      for (int i = 0; i < 8; i++) out.push_back((uint8_t)(mini >> (8 * i)));
      const size_t sh = 64 - written;
      mini = sh >= 64 ? 0 : (v >> sh);
      written = written + nb - 64;
    } else {
      mini |= (written < 64) ? (v << written) : 0;
      written += nb;
      if (written == 64) { for (int i = 0; i < 8; i++) out.push_back((uint8_t)(mini >> (8 * i))); written = 0; mini = 0; }
    }
  }
  void flush(std::vector<uint8_t>& out) {
    if (written > 0) { const size_t nbytes = (written + 7) / 8; for (size_t i = 0; i < nbytes; i++) out.push_back((uint8_t)(mini >> (8 * i))); written = 0; mini = 0; }
  }
};
static uint8_t num_bits(uint64_t n) { const uint8_t a = n ? (uint8_t)(64 - __builtin_clzll(n)) : 0; return a <= 56 ? a : 64; }
static void put64(std::vector<uint8_t>& o, uint64_t v) { for (int i = 0; i < 8; i++) o.push_back((uint8_t)(v >> (8 * i))); }
static void put32(std::vector<uint8_t>& o, uint32_t v) { for (int i = 0; i < 4; i++) o.push_back((uint8_t)(v >> (8 * i))); }
static uint64_t get64(const uint8_t* p) { uint64_t v = 0; for (int i = 0; i < 8; i++) v |= (uint64_t)p[i] << (8 * i); return v; }
static uint32_t get32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
static uint64_t extract_bits(const uint8_t* data, size_t len, size_t addr_bits, uint8_t nb) {  // :102-122
  const size_t ab = addr_bits / 8; const unsigned sh = addr_bits % 8;
  uint8_t buf[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (size_t i = 0; i < 8 && ab + i < len; i++) buf[i] = data[ab + i];
  const uint64_t v = get64(buf) >> sh;
  return v & ((1ull << nb) - 1ull);
}
static void flush_block(std::vector<Info>& b, std::vector<uint8_t>& metas, std::vector<uint8_t>& infos) {
  if (b.empty()) return;
  Packer bp;
  const Info ref = b[0], last = b.back();
  const uint64_t post_end = last.pe - ref.ps, pos_end = last.qe - ref.qs;
  uint32_t max_df = 0;
  for (size_t i = 1; i < b.size(); i++) { b[i].ps -= ref.ps; b[i].qs -= ref.qs; max_df = std::max(max_df, b[i].df); }
  const uint8_t dfb = num_bits(max_df), pb = num_bits(post_end), qb = num_bits(pos_end);
  put64(metas, infos.size());
  put32(metas, ref.df); put64(metas, ref.ps); put64(metas, ref.pe - ref.ps); put64(metas, ref.qs); put64(metas, ref.qe - ref.qs);
  metas.push_back(dfb); metas.push_back(pb); metas.push_back(qb);
  for (size_t i = 1; i < b.size(); i++) { bp.write(b[i].ps, pb, infos); bp.write(b[i].qs, qb, infos); bp.write(b[i].df, dfb, infos); }
  bp.write(post_end, pb, infos); bp.write(pos_end, qb, infos);
  bp.flush(infos);
  b.clear();
}
}  // namespace tis

// writes the store for n TermInfos; returns the byte length (call with out == NULL first)
ORC_API uint64_t orc_tis_write(const uint32_t* df, const uint64_t* ps, const uint64_t* pe, const uint64_t* qs, const uint64_t* qe,
                               uint64_t n, uint8_t* out) {
  std::vector<uint8_t> metas, infos; std::vector<tis::Info> blk;
  for (uint64_t i = 0; i < n; i++) {
    blk.push_back(tis::Info{df[i], ps[i], pe[i], qs[i], qe[i]});
    if (blk.size() >= 256) tis::flush_block(blk, metas, infos);
  }
  tis::flush_block(blk, metas, infos);
  std::vector<uint8_t> file;
  tis::put64(file, metas.size()); tis::put64(file, n);
  file.insert(file.end(), metas.begin(), metas.end());
  file.insert(file.end(), infos.begin(), infos.end());
  if (out) memcpy(out, file.data(), file.size());
  return file.size();
}
// TermInfoStore::get (:134-153)
ORC_API void orc_tis_get(const uint8_t* file, uint64_t len, uint64_t ord, uint32_t* df, uint64_t* ps, uint64_t* pe, uint64_t* qs, uint64_t* qe) {
  const uint64_t meta_len = tis::get64(file);
  const uint8_t* metas = file + 16; const uint8_t* infos = metas + meta_len; const size_t infos_len = (size_t)(len - 16 - meta_len);
  const uint8_t* m = metas + (ord / 256) * 47;
  const uint64_t off = tis::get64(m);
  const uint32_t rdf = tis::get32(m + 8); const uint64_t rps = tis::get64(m + 12), rpl = tis::get64(m + 20), rqs = tis::get64(m + 28), rql = tis::get64(m + 36);
  const uint8_t dfb = m[44], pb = m[45], qb = m[46];
  const uint64_t inner = ord % 256;
  if (inner == 0) { *df = rdf; *ps = rps; *pe = rps + rpl; *qs = rqs; *qe = rqs + rql; return; }
  const size_t nb = (size_t)dfb + pb + qb, a0 = nb * (inner - 1);
  const uint8_t* d = infos + off; const size_t dl = infos_len - (size_t)off;
  *ps = rps + tis::extract_bits(d, dl, a0, pb);
  *pe = rps + tis::extract_bits(d, dl, a0 + nb, pb);
  *qs = rqs + tis::extract_bits(d, dl, a0 + pb, qb);
  *qe = rqs + tis::extract_bits(d, dl, a0 + pb + nb, qb);
  *df = (uint32_t)tis::extract_bits(d, dl, a0 + pb + qb, dfb);
}
ORC_API uint64_t orc_tis_num_terms(const uint8_t* file) { return tis::get64(file + 8); }
// bitpacker KAT hook (term_info_store.rs:293-308): packs vals[i] at bits[i] and returns the byte length
ORC_API uint64_t orc_bitpack(const uint64_t* vals, const uint8_t* bits, uint32_t n, uint8_t* out) {
  tis::Packer bp; std::vector<uint8_t> o;
  for (uint32_t i = 0; i < n; i++) bp.write(vals[i], bits[i], o);
  bp.flush(o);
  memcpy(out, o.data(), o.size());
  return o.size();
}
ORC_API uint64_t orc_extract_bits(const uint8_t* data, uint64_t len, uint64_t addr_bits, uint8_t nb) { return tis::extract_bits(data, (size_t)len, (size_t)addr_bits, nb); }

// ---------------------------------------------------------------- numeric signals -------------
// PARITY UNPINNED: the reference has no test vectors for these transforms; tests/test_oracle_numeric.py pins hand-derived points.
// core/src/ranking/signals/core/non_text.rs: the value -> score part of every numeric CoreSignal's `compute`, written the way
// the reference writes it (one function per transform); `which` names the signal.
namespace numsig {
static double time_cache_calculation(double hours_since_update) { const double HALF_LIFE = 24.0 * 3.0; return HALF_LIFE / (hours_since_update + HALF_LIFE); }   // :44-47
static double score_timestamp(uint64_t page_timestamp, bool have_now, uint64_t now) {   // :25-42
  if (page_timestamp >= (have_now ? now : 0)) return 0.0;
  uint64_t d = now > page_timestamp ? now - page_timestamp : 0;   // saturating_sub
  if (d < 1) d = 1;
  const uint64_t hours = d / 3600;
  return hours < 3ull * 365 * 24 ? time_cache_calculation((double)hours) : 0.0;   // update_time_cache.get(hours).unwrap_or(0.0)
}
static double score_rank(double rank) { const double v = 10.0 - std::log(1.0 + rank) / std::log(8.0); return v > 0.0 ? v : 0.0; }   // :50-59, f64::log(base)
static double score_inverse(double x) { return 1.0 / (x + 1.0); }   // score_trackers / score_digits / score_slashes :61-74
static double score_link_density(double x) { return x > 0.5 ? 0.0 : 1.0 - x; }   // :76-83
}  // namespace numsig
// which: 0 HostCentrality/PageCentrality, 1 *CentralityRank, 2 IsHomepage, 3 HasAds, 4 TrackerScore/UrlDigits/UrlSlashes, 5 FetchTimeMs,
//        6 UpdateTimestamp (now < 0: no current timestamp), 7 LinkDensity, 8 Region (counts NULL: no RegionCount; selected < 0: none / All)
ORC_API void orc_numeric_scores(uint32_t which, const uint64_t* raw_u, const double* raw_f, const uint8_t* raw_b, uint32_t n, int64_t now,
                                const int64_t* region_counts, uint32_t n_regions, uint64_t region_total, int64_t selected, double* out) {
  for (uint32_t d = 0; d < n; d++) {
    double s = 0.0;
    switch (which) {
      case 0: s = raw_f[d]; break;
      case 1: s = numsig::score_rank((double)raw_u[d]); break;
      case 2: s = raw_b[d] ? 1.0 : 0.0; break;
      case 3: s = !raw_b[d] ? 1.0 : 0.0; break;
      case 4: s = numsig::score_inverse((double)raw_u[d]); break;
      case 5: { const uint64_t x = raw_u[d]; s = x >= 1000 ? 0.0 : 1.0 / ((double)x + 1.0); break; }   // fetch_time_ms_cache, computer/mod.rs:257-259
      case 6: s = numsig::score_timestamp(raw_u[d], now >= 0, now >= 0 ? (uint64_t)now : 0); break;
      case 7: s = numsig::score_link_density(raw_f[d]); break;
      case 8: {   // score_region :85-101 + RegionCount::score (webpage/region.rs:219-227); a negative count = None
        if (region_counts) {
          const uint64_t id = raw_u[d];
          const double boost = (selected >= 0 && (uint64_t)selected == id) ? 50.0 : 0.0;
          double share = 0.0;
          if (id < n_regions && region_counts[id] >= 0) share = (double)region_counts[id] / (double)region_total;
          s = boost + share;
        }
        break;
      }
    }
    out[d] = s;
  }
}
