// lambdamart.cu -- Stract's LambdaMART model (see stract_b200_lambdamart.h): the reference's text format parsed and validated on
// the host, a batched tree-ensemble kernel on the device.
//
// Device layout of a model (one blob of 16-byte units, trees contiguous in tree order):
//   tree t   its internal records (the nodes some path from the root reaches, depth-first preorder, root first), then its leaf
//            values as f64 with the reference's offset already added (leaf + (|min| + 1.0), in f64 on the host)
//   record   { f64 threshold, u32 left, u32 right }: a child is a record index, or a leaf index with bit 31 set; bits 24..30 of
//            `left` hold the record's feature as a column of the CTA's feature tile
//   tree_tab per tree { first record, first leaf } in f64 words from the start of the blob
//   chunks   runs of consecutive trees that fit the shared tree buffer together; a tree larger than the buffer is a chunk of
//            its own that is walked from global memory
// k_lambdamart: one thread owns one document of a TILE-document CTA.  The CTA stages its documents' used feature columns in
// shared memory as [column][TILE] (thread t reads word t of a column: the bank depends on t alone, so any mix of columns
// across a warp is conflict-free), then streams the chunks through the tree buffer.  Each thread walks two trees at a time
// (independent loads in flight) and adds their leaves to one f64 register in tree order, so the sum is the reference's
// sequential sum; one division at the end.
#include "common.cuh"
#include "../../include/stract_b200_lambdamart.h"

#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdlib>
#include <limits>
#include <string>
#include <vector>

namespace sb200 {
namespace lm {

constexpr int TILE = 128;                 // documents (threads) per CTA
constexpr uint32_t BUF_UNITS = 2048;      // shared tree buffer: 32 KB of 16-byte units
constexpr uint32_t LEAF_BIT = 0x80000000u;
constexpr uint32_t IDX_MASK = 0x00FFFFFFu;
constexpr uint32_t MAX_SLOTS = 1u << 24;
constexpr uint8_t NO_COL = 0xFF;

// SignalEnum in declaration order (ranking/signals/mod.rs:108-155), serde snake_case
static const char* const SIGNAL_NAMES[SB200_SIGNAL_ENUM_COUNT] = {
    "bm25_f", "bm25_title", "title_coverage", "bm25_title_bigrams", "bm25_title_trigrams", "bm25_clean_body",
    "clean_body_coverage", "bm25_clean_body_bigrams", "bm25_clean_body_trigrams", "bm25_stemmed_title",
    "bm25_stemmed_clean_body", "bm25_all_body", "bm25_keywords", "bm25_backlink_text", "idf_sum_url", "idf_sum_site",
    "idf_sum_domain", "idf_sum_site_no_tokenizer", "idf_sum_domain_no_tokenizer", "idf_sum_domain_name_no_tokenizer",
    "idf_sum_domain_if_homepage", "idf_sum_domain_name_if_homepage_no_tokenizer", "idf_sum_domain_if_homepage_no_tokenizer",
    "idf_sum_title_if_homepage", "cross_encoder_snippet", "cross_encoder_title", "host_centrality", "host_centrality_rank",
    "page_centrality", "page_centrality_rank", "is_homepage", "fetch_time_ms", "update_timestamp", "tracker_score", "region",
    "query_centrality", "inbound_similarity", "lambda_mart", "url_digits", "url_slashes", "link_density",
    "title_embedding_similarity", "keyword_embedding_similarity", "has_ads", "min_title_slop", "min_clean_body_slop"};

struct Record { double thr; uint32_t left, right; };
static_assert(sizeof(Record) == 16, "one record is one 16-byte unit");

__global__ void __launch_bounds__(TILE) k_lambdamart(const double* __restrict__ feats, uint64_t n_docs, const uint4* __restrict__ blob,
                                                     const uint32_t* __restrict__ tree_tab, const uint4* __restrict__ chunks, uint32_t n_chunks,
                                                     uint32_t n_trees, const uint8_t* __restrict__ colmap, uint32_t n_used,
                                                     double* __restrict__ out) {
  SB_DYN_SMEM(smem);
  __shared__ uint8_t scol[SB200_SIGNAL_ENUM_COUNT];
  double* sf = (double*)smem;                              // [n_used][TILE]
  uint4* sbuf = (uint4*)(smem + (size_t)n_used * TILE * 8);  // BUF_UNITS units
  const uint32_t tid = threadIdx.x;
  const uint64_t d0 = (uint64_t)blockIdx.x * TILE;
  const uint32_t nd = n_docs - d0 < (uint64_t)TILE ? (uint32_t)(n_docs - d0) : (uint32_t)TILE;
  if (tid < SB200_SIGNAL_ENUM_COUNT) scol[tid] = colmap[tid];
  __syncthreads();
  // the tile's rows are one contiguous run of nd * 46 f64: read it coalesced, keep the used columns
  const double* rows = feats + d0 * SB200_SIGNAL_ENUM_COUNT;
  for (uint32_t i = tid; i < nd * SB200_SIGNAL_ENUM_COUNT; i += TILE) {
    const uint32_t r = i / SB200_SIGNAL_ENUM_COUNT, c = i - r * SB200_SIGNAL_ENUM_COUNT;
    const uint8_t s = scol[c];
    if (s != NO_COL) sf[s * TILE + r] = __ldg(rows + i);
  }
  const double* myf = sf + tid;
  double acc = 0.0;
  for (uint32_t c = 0; c < n_chunks; c++) {
    const uint4 ch = __ldg(chunks + c);   // first tree, end tree, first unit, end unit | global flag
    const bool global = (ch.w & LEAF_BIT) != 0;
    const uint32_t u0 = ch.z, u1 = ch.w & ~LEAF_BIT;
    __syncthreads();                      // the previous chunk's walks are done (first pass: the feature tile is written)
    if (!global) {
      for (uint32_t u = u0 + tid; u < u1; u += TILE) sbuf[u - u0] = __ldg(blob + u);
      __syncthreads();
    }
    const uint4* base = global ? blob : sbuf;
    const uint32_t sub = global ? 0u : 2u * u0;   // f64 words
    if (tid >= nd) continue;
    auto step = [&](uint32_t rec0, uint32_t& node, uint32_t leaf0, double& leaf) -> bool {
      const uint4 r = base[(rec0 >> 1) + node];
      const double thr = __longlong_as_double((long long)(((unsigned long long)r.y << 32) | r.x));
      const double v = myf[((r.z >> 24) & 0x7Fu) * TILE];
      const uint32_t nxt = v <= thr ? r.z : r.w;
      if (nxt & LEAF_BIT) {
        const uint32_t li = leaf0 + (nxt & IDX_MASK);
        const uint4 lw = base[li >> 1];
        const uint32_t lo = (li & 1u) ? lw.z : lw.x, hi = (li & 1u) ? lw.w : lw.y;
        leaf = __longlong_as_double((long long)(((unsigned long long)hi << 32) | lo));
        return true;
      }
      node = nxt & IDX_MASK;
      return false;
    };
    uint32_t t = ch.x;
    for (; t + 1 < ch.y; t += 2) {   // two independent walks in flight, leaves added in tree order
      const uint32_t ra = __ldg(tree_tab + 2 * t) - sub, la0 = __ldg(tree_tab + 2 * t + 1) - sub;
      const uint32_t rb = __ldg(tree_tab + 2 * t + 2) - sub, lb0 = __ldg(tree_tab + 2 * t + 3) - sub;
      uint32_t na = 0, nb = 0;
      double la = 0.0, lb = 0.0;
      bool da = false, db = false;
      while (!(da && db)) {
        if (!da) da = step(ra, na, la0, la);
        if (!db) db = step(rb, nb, lb0, lb);
      }
      acc = acc + la;
      acc = acc + lb;
    }
    if (t < ch.y) {
      const uint32_t ra = __ldg(tree_tab + 2 * t) - sub, la0 = __ldg(tree_tab + 2 * t + 1) - sub;
      uint32_t na = 0;
      double la = 0.0;
      while (!step(ra, na, la0, la)) {}
      acc = acc + la;
    }
  }
  if (tid < nd) out[d0 + tid] = acc / (double)n_trees;
}

// ---- host: the reference's parser -------------------------------------------------------------------------------------------
struct Error { std::string msg; };

static bool valid_utf8(const unsigned char* s, size_t n) {
  size_t i = 0;
  while (i < n) {
    const unsigned c = s[i];
    if (c < 0x80) { i++; continue; }
    int len; unsigned cp, lo;
    if ((c & 0xE0) == 0xC0) { len = 2; cp = c & 0x1F; lo = 0x80; }
    else if ((c & 0xF0) == 0xE0) { len = 3; cp = c & 0x0F; lo = 0x800; }
    else if ((c & 0xF8) == 0xF0) { len = 4; cp = c & 0x07; lo = 0x10000; }
    else return false;
    if (i + len > n) return false;
    for (int k = 1; k < len; k++) {
      if ((s[i + k] & 0xC0) != 0x80) return false;
      cp = (cp << 6) | (s[i + k] & 0x3F);
    }
    if (cp < lo || cp > 0x10FFFF || (cp >= 0xD800 && cp <= 0xDFFF)) return false;
    i += len;
  }
  return true;
}

// str::lines: split on '\n', one '\r' before it dropped, no empty line after a final '\n'
static std::vector<std::string> rust_lines(const std::string& s) {
  std::vector<std::string> out;
  size_t i = 0;
  while (i < s.size()) {
    const size_t j = s.find('\n', i);
    if (j == std::string::npos) { out.push_back(s.substr(i)); break; }
    std::string l = s.substr(i, j - i);
    if (!l.empty() && l.back() == '\r') l.pop_back();
    out.push_back(std::move(l));
    i = j + 1;
  }
  return out;
}

static std::string join(const std::vector<std::string>& v, size_t a, size_t b) {
  std::string s;
  for (size_t i = a; i < b; i++) { if (i > a) s += '\n'; s += v[i]; }
  return s;
}

static std::vector<std::string> split_space(const std::string& s) {
  std::vector<std::string> out;
  size_t i = 0;
  for (;;) {
    const size_t j = s.find(' ', i);
    if (j == std::string::npos) { out.push_back(s.substr(i)); return out; }
    out.push_back(s.substr(i, j - i));
    i = j + 1;
  }
}

// char::is_whitespace
static bool rust_ws(uint32_t cp) {
  return (cp >= 0x09 && cp <= 0x0D) || cp == 0x20 || cp == 0x85 || cp == 0xA0 || cp == 0x1680 || (cp >= 0x2000 && cp <= 0x200A) ||
         cp == 0x2028 || cp == 0x2029 || cp == 0x202F || cp == 0x205F || cp == 0x3000;
}

// str::trim (Unicode White_Space) of valid UTF-8 compared with `want`
static bool trim_equals(const std::string& s, const char* want) {
  std::vector<uint32_t> cps;
  std::vector<size_t> at;
  for (size_t i = 0; i < s.size();) {
    const unsigned char c = (unsigned char)s[i];
    const int len = c < 0x80 ? 1 : (c & 0xE0) == 0xC0 ? 2 : (c & 0xF0) == 0xE0 ? 3 : 4;
    uint32_t cp = len == 1 ? c : len == 2 ? (c & 0x1F) : len == 3 ? (c & 0x0F) : (c & 0x07);
    for (int k = 1; k < len; k++) cp = (cp << 6) | ((unsigned char)s[i + k] & 0x3F);
    cps.push_back(cp); at.push_back(i);
    i += len;
  }
  at.push_back(s.size());
  size_t a = 0, b = cps.size();
  while (a < b && rust_ws(cps[a])) a++;
  while (b > a && rust_ws(cps[b - 1])) b--;
  return s.compare(at[a], at[b] - at[a], want) == 0;
}

static bool all_digits(const std::string& s, size_t from) {
  if (from >= s.size()) return false;
  for (size_t i = from; i < s.size(); i++) if (s[i] < '0' || s[i] > '9') return false;
  return true;
}

// <usize as FromStr>: optional '+', ASCII digits, no overflow
static uint64_t parse_usize(const std::string& s) {
  const size_t a = (!s.empty() && s[0] == '+') ? 1 : 0;
  if (!all_digits(s, a)) throw Error{"ParseInt: ParseInt error: cannot parse `" + s + "` as usize"};
  uint64_t v = 0;
  for (size_t i = a; i < s.size(); i++) {
    const uint64_t d = (uint64_t)(s[i] - '0');
    if (v > (UINT64_MAX - d) / 10) throw Error{"ParseInt: ParseInt error: `" + s + "` overflows usize"};
    v = v * 10 + d;
  }
  return v;
}

// <i32 as FromStr>: optional sign, ASCII digits, in range
static int64_t parse_i32(const std::string& s) {
  const bool neg = !s.empty() && s[0] == '-';
  const size_t a = (!s.empty() && (s[0] == '+' || s[0] == '-')) ? 1 : 0;
  if (!all_digits(s, a)) throw Error{"ParseInt: ParseInt error: cannot parse `" + s + "` as i32"};
  int64_t v = 0;
  for (size_t i = a; i < s.size(); i++) {
    v = v * 10 + (s[i] - '0');
    if (v > 2147483648ll) throw Error{"ParseInt: ParseInt error: `" + s + "` is out of the range of i32"};
  }
  if (!neg && v > 2147483647ll) throw Error{"ParseInt: ParseInt error: `" + s + "` is out of the range of i32"};
  return neg ? -v : v;
}

static bool ieq(const std::string& s, size_t a, const char* w) {
  const size_t n = strlen(w);
  if (s.size() - a != n) return false;
  for (size_t i = 0; i < n; i++) if (tolower((unsigned char)s[a + i]) != w[i]) return false;
  return true;
}

// <f64 as FromStr>: [+-]? (digits [. digits?] | . digits) ([eE] [+-]? digits)?  or  [+-]? (inf | infinity | nan), case-insensitive;
// no whitespace, underscores, hex or nan(...) forms.  Decimal forms are correctly rounded, like strtod.
static double parse_f64(const std::string& s) {
  const bool neg = !s.empty() && s[0] == '-';
  const size_t a = (!s.empty() && (s[0] == '+' || s[0] == '-')) ? 1 : 0;
  if (ieq(s, a, "inf") || ieq(s, a, "infinity")) return neg ? -HUGE_VAL : HUGE_VAL;
  if (ieq(s, a, "nan")) return neg ? -std::numeric_limits<double>::quiet_NaN() : std::numeric_limits<double>::quiet_NaN();
  size_t i = a, mant = 0;
  while (i < s.size() && isdigit((unsigned char)s[i])) { i++; mant++; }
  if (i < s.size() && s[i] == '.') { i++; while (i < s.size() && isdigit((unsigned char)s[i])) { i++; mant++; } }
  bool ok = mant > 0;
  if (ok && i < s.size() && (s[i] == 'e' || s[i] == 'E')) {
    i++;
    if (i < s.size() && (s[i] == '+' || s[i] == '-')) i++;
    size_t e = 0;
    while (i < s.size() && isdigit((unsigned char)s[i])) { i++; e++; }
    ok = e > 0;
  }
  if (!ok || i != s.size()) throw Error{"ParseFloat: ParseFloat error: invalid float literal `" + s + "`"};
  return strtod(s.c_str(), nullptr);
}

struct Child { bool some = false, leaf = false; uint64_t idx = 0; };
struct Slot { int feature = -1; double thr = 0.0, leaf = 0.0; Child left, right; };
struct Tree { std::vector<Slot> nodes; };

static Child parse_child(const std::string& tok) {
  const int64_t c = parse_i32(tok);
  Child ch; ch.some = true;
  if (c < 0) { ch.leaf = true; ch.idx = (uint64_t)(-c) - 1; }
  else ch.idx = (uint64_t)c;
  return ch;
}

static Tree parse_tree(const std::string& s, const std::vector<int>& header, size_t t) {
  std::vector<int> feats;
  std::vector<double> thr, leaves;
  std::vector<Child> lefts, rights;
  for (const std::string& line : rust_lines(s)) {
    const size_t eq = line.find('=');
    if (eq == std::string::npos) continue;
    const std::string key = line.substr(0, eq), value = line.substr(eq + 1);
    if (key == "split_feature") {
      for (const std::string& tok : split_space(value)) {
        const uint64_t i = parse_usize(tok);
        if (i >= header.size())
          throw Error{"panic: tree " + std::to_string(t) + ": split_feature " + std::to_string(i) + " is out of bounds for " +
                      std::to_string(header.size()) + " header features"};
        feats.push_back(header[i]);
      }
    } else if (key == "threshold") {
      for (const std::string& tok : split_space(value)) thr.push_back(parse_f64(tok));
    } else if (key == "leaf_value") {
      for (const std::string& tok : split_space(value)) leaves.push_back(parse_f64(tok));
    } else if (key == "left_child") {
      for (const std::string& tok : split_space(value)) lefts.push_back(parse_child(tok));
    } else if (key == "right_child") {
      for (const std::string& tok : split_space(value)) rights.push_back(parse_child(tok));
    }
  }
  // offset = |fold(cur < v ? cur : v)| + 1.0, every leaf shifted by it (f64, as the reference adds it)
  Tree tr;
  if (!leaves.empty()) {
    double m = leaves[0];
    for (size_t i = 1; i < leaves.size(); i++) m = m < leaves[i] ? m : leaves[i];
    const double off = std::fabs(m) + 1.0;
    tr.nodes.resize(leaves.size());
    for (size_t i = 0; i < leaves.size(); i++) tr.nodes[i].leaf = leaves[i] + off;
  }
  const size_t n = tr.nodes.size();
  auto fits = [&](size_t k, const char* what) {
    if (k > n)
      throw Error{"panic: tree " + std::to_string(t) + ": " + std::to_string(k) + " " + what + " entries for " + std::to_string(n) +
                  " node slots (index out of bounds)"};
  };
  fits(feats.size(), "split_feature");
  for (size_t i = 0; i < feats.size(); i++) tr.nodes[i].feature = feats[i];
  fits(thr.size(), "threshold");
  for (size_t i = 0; i < thr.size(); i++) tr.nodes[i].thr = thr[i];
  fits(lefts.size(), "left_child");
  for (size_t i = 0; i < lefts.size(); i++) tr.nodes[i].left = lefts[i];
  fits(rights.size(), "right_child");
  for (size_t i = 0; i < rights.size(); i++) tr.nodes[i].right = rights[i];
  return tr;
}

static std::vector<Tree> parse_model(const std::string& text, std::vector<int>& header) {
  const std::vector<std::string> lines = rust_lines(text);
  size_t end_header = 0;
  while (end_header < lines.size() && !lines[end_header].empty()) end_header++;
  if (end_header == lines.size()) throw Error{"panic: no empty line ends the header (Option::unwrap on None)"};
  for (const std::string& lin : rust_lines(join(lines, 0, end_header))) {
    const size_t eq = lin.find('=');
    if (eq == std::string::npos || lin.compare(0, eq, "feature_names") != 0) continue;
    for (const std::string& name : split_space(lin.substr(eq + 1))) {
      int f = -1;
      for (int k = 0; k < SB200_SIGNAL_ENUM_COUNT; k++) if (name == SIGNAL_NAMES[k]) { f = k; break; }
      if (f < 0) throw Error{"UnknownSignal: Unknown signal: " + name};
      header.push_back(f);
    }
  }
  if (header.empty()) throw Error{"NoFeatures: no features found"};
  size_t end_trees = 0;
  while (end_trees < lines.size() && !trim_equals(lines[end_trees], "end of trees")) end_trees++;
  if (end_trees == lines.size()) throw Error{"NoEndOfTrees: couldn't find end of trees"};
  std::vector<Tree> trees;
  for (size_t start = end_header + 1; start < end_trees;) {
    size_t end = start;
    while (end < lines.size() && !lines[end].empty()) end++;
    if (end == lines.size())
      throw Error{"panic: tree " + std::to_string(trees.size()) + ": no empty line ends the tree (Option::unwrap on None)"};
    trees.push_back(parse_tree(join(lines, start, end), header, trees.size()));
    start = end + 2;
  }
  return trees;
}

// ---- host: load-time refusal and flattening ---------------------------------------------------------------------------------
// Every path from the root must end at a leaf.  A left edge exists unless the threshold is NaN (value <= NaN never holds); the
// right edge always exists (a NaN value goes right).  Records are numbered in depth-first preorder of the reachable nodes; bits
// 24..30 of `left` hold the SignalEnum ordinal until build() maps it to a feature-tile column.
struct Flat {
  std::vector<Record> recs;
  uint32_t depth = 0;
};

static Flat flatten(const Tree& tr, size_t t) {
  const size_t n = tr.nodes.size();
  const std::string T = "tree " + std::to_string(t);
  if (n == 0) throw Error{"panic: " + T + " has no node slots (index out of bounds: nodes[0])"};
  if (n >= MAX_SLOTS) throw Error{"range: " + T + " has " + std::to_string(n) + " node slots, at most 2^24 - 1 are supported"};
  std::vector<int> state(n, 0);          // 0 unseen, 1 on the stack, 2 done
  std::vector<uint32_t> rec_of(n, 0), depth(n, 0);
  Flat f;
  struct Frame { uint32_t node; int edge; };
  std::vector<Frame> st{{0, 0}};
  auto visit = [&](uint32_t i) {
    const Slot& s = tr.nodes[i];
    if (s.feature < 0) throw Error{"panic: " + T + " node " + std::to_string(i) + " has no feature (LeafNotFound unwrapped)"};
    if (!std::isnan(s.thr) && !s.left.some)
      throw Error{"panic: " + T + " node " + std::to_string(i) + " has no left child (LeafNotFound unwrapped)"};
    if (!s.right.some) throw Error{"panic: " + T + " node " + std::to_string(i) + " has no right child (LeafNotFound unwrapped)"};
    state[i] = 1;
    rec_of[i] = (uint32_t)f.recs.size();
    f.recs.push_back(Record{s.thr, 0, 0});
  };
  visit(0);
  while (!st.empty()) {
    Frame& fr = st.back();
    const uint32_t i = fr.node;
    const Slot& s = tr.nodes[i];
    if (fr.edge == 2) {
      uint32_t d = 0;
      for (int e = 0; e < 2; e++) {
        const Child& c = e ? s.right : s.left;
        if (e == 0 && std::isnan(s.thr)) continue;
        if (!c.leaf) d = std::max(d, depth[c.idx]);
      }
      depth[i] = d + 1;
      state[i] = 2;
      st.pop_back();
      continue;
    }
    const int e = fr.edge++;
    if (e == 0 && std::isnan(s.thr)) continue;
    const Child& c = e ? s.right : s.left;
    if (c.idx >= n)
      throw Error{"panic: " + T + " node " + std::to_string(i) + ": child index " + std::to_string(c.idx) + " is out of bounds for " +
                  std::to_string(n) + " node slots"};
    if (c.leaf || state[c.idx] == 2) continue;
    if (state[c.idx] == 1) throw Error{"loops forever: " + T + " has a cycle through node " + std::to_string(c.idx)};
    visit((uint32_t)c.idx);
    st.push_back(Frame{(uint32_t)c.idx, 0});
  }
  for (size_t i = 0; i < n; i++) {
    if (state[i] != 2) continue;
    const Slot& s = tr.nodes[i];
    auto enc = [&](const Child& c, bool taken) -> uint32_t {
      if (!taken) return LEAF_BIT;                  // the left edge of a NaN threshold: never followed
      return c.leaf ? (LEAF_BIT | (uint32_t)c.idx) : rec_of[c.idx];
    };
    Record& r = f.recs[rec_of[i]];
    r.left = enc(s.left, !std::isnan(s.thr)) | ((uint32_t)s.feature << 24);
    r.right = enc(s.right, true);
  }
  f.depth = depth[0];
  return f;
}

}  // namespace lm
}  // namespace sb200

struct sb200_lambdamart {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, evk0 = nullptr, evk1 = nullptr;
  uint32_t n_trees = 0, n_used = 0, max_depth = 0;
  uint64_t n_internal = 0, n_leaves = 0;
  std::vector<uint32_t> features;        // header features as SignalEnum ordinals
  std::vector<uint4> h_chunks;
  sb200::DevBuf<uint4> blob, chunks;
  sb200::DevBuf<uint32_t> tree_tab;     // per tree { first record, first leaf } in f64 words
  sb200::DevBuf<uint8_t> colmap;
  sb200::DevBuf<double> in, out;         // scratch for host inputs / outputs, grown on demand
  ~sb200_lambdamart() {
    blob.release(); chunks.release(); tree_tab.release(); colmap.release(); in.release(); out.release();
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (evk0) cudaEventDestroy(evk0);
    if (evk1) cudaEventDestroy(evk1);
    if (stream) cudaStreamDestroy(stream);
  }
};

namespace sb200 {
namespace lm {
static size_t smem_bytes(uint32_t n_used) { return (size_t)n_used * TILE * 8 + (size_t)BUF_UNITS * 16; }

static int build(const char* text, uint64_t len, sb200_lambdamart* m) {
  std::vector<int> header;
  if (!valid_utf8((const unsigned char*)text, len)) SB_FAIL(SB200_EFORMAT, "Io: stream did not contain valid UTF-8");
  std::vector<Tree> trees;
  std::vector<Flat> flats;
  std::vector<int> colmap(SB200_SIGNAL_ENUM_COUNT, NO_COL);
  try {
    trees = parse_model(std::string(text, len), header);
    for (size_t t = 0; t < trees.size(); t++) flats.push_back(flatten(trees[t], t));
  } catch (const Error& e) {
    if (e.msg.compare(0, 6, "range:") == 0) SB_FAIL(SB200_ERANGE, "%s", e.msg.c_str() + 7);
    SB_FAIL(SB200_EFORMAT, "%s", e.msg.c_str());
  }
  // the feature tile holds the columns some record reads, in SignalEnum order
  std::vector<char> used(SB200_SIGNAL_ENUM_COUNT, 0);
  for (const Flat& f : flats) for (const Record& r : f.recs) used[(r.left >> 24) & 0x7Fu] = 1;
  for (int c = 0; c < SB200_SIGNAL_ENUM_COUNT; c++) if (used[c]) colmap[c] = (int)m->n_used++;
  for (Flat& f : flats) for (Record& r : f.recs) r.left = (r.left & ~(0x7Fu << 24)) | ((uint32_t)colmap[(r.left >> 24) & 0x7Fu] << 24);
  for (int f : header) m->features.push_back((uint32_t)f);
  m->n_trees = (uint32_t)trees.size();
  // the blob: per tree records, then leaves padded to a whole unit
  std::vector<uint4> blob;
  std::vector<uint32_t> tab;
  std::vector<uint64_t> tree_unit;
  for (size_t t = 0; t < trees.size(); t++) {
    const Flat& f = flats[t];
    const uint64_t u = blob.size();
    tree_unit.push_back(u);
    const uint64_t nl = trees[t].nodes.size();
    if ((u + f.recs.size()) * 2 + nl > 0xFFFFFFFFull) SB_FAIL(SB200_ERANGE, "model above 32 GB");
    tab.push_back((uint32_t)(u * 2));
    tab.push_back((uint32_t)((u + f.recs.size()) * 2));
    for (const Record& r : f.recs) { uint4 x; memcpy(&x, &r, 16); blob.push_back(x); }
    std::vector<double> lv(nl + (nl & 1), 0.0);
    for (size_t i = 0; i < nl; i++) lv[i] = trees[t].nodes[i].leaf;
    for (size_t i = 0; i < lv.size(); i += 2) { uint4 x; memcpy(&x, &lv[i], 16); blob.push_back(x); }
    m->n_internal += f.recs.size();
    m->n_leaves += nl;
    m->max_depth = std::max(m->max_depth, f.depth);
  }
  tree_unit.push_back(blob.size());
  for (uint32_t t = 0; t < m->n_trees;) {   // greedy runs of whole trees that fit the buffer; a larger tree alone, from global memory
    uint32_t e = t;
    while (e < m->n_trees && tree_unit[e + 1] - tree_unit[t] <= BUF_UNITS) e++;
    const bool global = e == t;
    if (global) e = t + 1;
    m->h_chunks.push_back(make_uint4(t, e, (uint32_t)tree_unit[t], (uint32_t)tree_unit[e] | (global ? LEAF_BIT : 0u)));
    t = e;
  }
  if (blob.size() >= LEAF_BIT) SB_FAIL(SB200_ERANGE, "model above 32 GB");
  std::vector<uint8_t> cm(colmap.begin(), colmap.end());
  SB_TRY(m->blob.alloc(blob.size()));
  SB_TRY(m->tree_tab.alloc(tab.size()));
  SB_TRY(m->chunks.alloc(m->h_chunks.size()));
  SB_TRY(m->colmap.alloc(cm.size()));
  if (!blob.empty()) SB_CUDA(cudaMemcpy(m->blob.p, blob.data(), blob.size() * 16, cudaMemcpyHostToDevice));
  if (!tab.empty()) SB_CUDA(cudaMemcpy(m->tree_tab.p, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice));
  if (!m->h_chunks.empty()) SB_CUDA(cudaMemcpy(m->chunks.p, m->h_chunks.data(), m->h_chunks.size() * 16, cudaMemcpyHostToDevice));
  SB_CUDA(cudaMemcpy(m->colmap.p, cm.data(), cm.size(), cudaMemcpyHostToDevice));
  return SB200_OK;
}
}  // namespace lm
}  // namespace sb200

extern "C" {

int sb200_lambdamart_load(const char* text, uint64_t len, sb200_lambdamart** out) {
  using namespace sb200;
  if (!out || (!text && len)) SB_FAIL(SB200_EINVAL, "NULL argument");
  *out = nullptr;
  sb200_lambdamart* m = new (std::nothrow) sb200_lambdamart();
  if (!m) SB_FAIL(SB200_ENOMEM, "host allocation failed");
  int rc = cudaGetDevice(&m->device) == cudaSuccess ? SB200_OK : SB200_ECUDA;
  if (rc != SB200_OK) set_error("cudaGetDevice failed");
  if (rc == SB200_OK && (cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreate(&m->ev0) != cudaSuccess ||
                         cudaEventCreate(&m->ev1) != cudaSuccess || cudaEventCreate(&m->evk0) != cudaSuccess ||
                         cudaEventCreate(&m->evk1) != cudaSuccess)) {
    set_error("stream / event creation failed");
    rc = SB200_ECUDA;
  }
  if (rc == SB200_OK) rc = lm::build(text ? text : "", len, m);
  if (rc != SB200_OK) { delete m; return rc; }
  *out = m;
  return SB200_OK;
}

void sb200_lambdamart_destroy(sb200_lambdamart* m) {
  if (!m) return;
  cudaSetDevice(m->device);
  delete m;
}

int sb200_lambdamart_get_info(const sb200_lambdamart* m, sb200_lambdamart_info* info) {
  if (!m || !info) SB_FAIL(SB200_EINVAL, "NULL argument");
  memset(info, 0, sizeof(*info));
  info->n_trees = m->n_trees;
  info->n_features = (uint32_t)m->features.size();
  info->n_internal = m->n_internal;
  info->n_leaves = m->n_leaves;
  info->max_depth = m->max_depth;
  info->device_bytes = m->blob.bytes() + m->tree_tab.bytes() + m->chunks.bytes() + m->colmap.bytes() + m->in.bytes() + m->out.bytes();
  return SB200_OK;
}

int sb200_lambdamart_features(const sb200_lambdamart* m, uint32_t* ordinals, uint32_t cap) {
  if (!m || (cap && !ordinals)) SB_FAIL(SB200_EINVAL, "NULL argument");
  for (uint32_t i = 0; i < cap && i < m->features.size(); i++) ordinals[i] = m->features[i];
  return SB200_OK;
}

int sb200_lambdamart_predict(sb200_lambdamart* m, const double* features, uint64_t n_docs, double* out, sb200_lambdamart_stats* stats) {
  using namespace sb200;
  using namespace sb200::lm;
  if (!m) SB_FAIL(SB200_EINVAL, "NULL model");
  if (n_docs && (!features || !out)) SB_FAIL(SB200_EINVAL, "NULL features / out");
  if (n_docs > (uint64_t)0x7FFFFFFF * TILE) SB_FAIL(SB200_ERANGE, "n_docs %llu above the grid limit", (unsigned long long)n_docs);
  if (stats) memset(stats, 0, sizeof(*stats));
  if (n_docs == 0) return SB200_OK;
  SB_CUDA(cudaSetDevice(m->device));
  NvtxRange nvtx("lambdamart_predict");
  const size_t in_bytes = (size_t)n_docs * SB200_SIGNAL_ENUM_COUNT * 8;
  SB_CUDA(cudaEventRecord(m->ev0, m->stream));
  const double* d_in = features;
  if (!is_device_ptr(features)) {
    if (m->in.n < n_docs * SB200_SIGNAL_ENUM_COUNT) SB_TRY(m->in.alloc(n_docs * SB200_SIGNAL_ENUM_COUNT));
    SB_CUDA(cudaMemcpyAsync(m->in.p, features, in_bytes, cudaMemcpyHostToDevice, m->stream));
    d_in = m->in.p;
  }
  double* d_out = out;
  const bool host_out = !is_device_ptr(out);
  if (host_out) {
    if (m->out.n < n_docs) SB_TRY(m->out.alloc(n_docs));
    d_out = m->out.p;
  }
  const size_t smem = smem_bytes(m->n_used);
#ifndef SB200_EMU
  SB_CUDA(cudaFuncSetAttribute(k_lambdamart, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
#endif
  SB_CUDA(cudaEventRecord(m->evk0, m->stream));
  SB_LAUNCH(k_lambdamart, div_up(n_docs, TILE), TILE, smem, m->stream, d_in, n_docs, m->blob.p, m->tree_tab.p, m->chunks.p,
            (uint32_t)m->h_chunks.size(), m->n_trees, m->colmap.p, m->n_used, d_out);
  SB_CHECK_LAUNCH();
  SB_CUDA(cudaEventRecord(m->evk1, m->stream));
  if (host_out) SB_CUDA(cudaMemcpyAsync(out, d_out, (size_t)n_docs * 8, cudaMemcpyDeviceToHost, m->stream));
  SB_CUDA(cudaEventRecord(m->ev1, m->stream));
  SB_CUDA(cudaStreamSynchronize(m->stream));
  if (stats) {
    stats->docs = n_docs;
    SB_CUDA(cudaEventElapsedTime(&stats->ms, m->ev0, m->ev1));
    SB_CUDA(cudaEventElapsedTime(&stats->kernel_ms, m->evk0, m->evk1));
  }
  return SB200_OK;
}

}  // extern "C"
