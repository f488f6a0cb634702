/* stract_b200_bm25.h -- C ABI of hot path 2: BM25 posting-list scoring + top-k collection over
 * tantivy-format posting lists (part of libstract_b200.so; conventions as in stract_b200.h).
 *
 * Replaces, per segment (paths relative to /root/reference/crates):
 *   (A) tantivy-native top-k:  TopDocs::collect_segment -> Weight::for_each_pruning -> Intersection /
 *       block_wand -> TermScorer::score -> TopNComputer
 *         tantivy/src/collector/top_score_collector.rs:385-413,501-564, tantivy/src/query/weight.rs:47-60,
 *         tantivy/src/query/intersection.rs:14-160, tantivy/src/query/boolean_query/block_wand.rs:148-214,
 *         tantivy/src/query/term_query/term_scorer.rs:119-123, tantivy/src/query/bm25.rs:182-196
 *   (B) Stract's recall stage: TweakedScoreTopCollector + InitialSegmentScoreTweaker::score
 *       (Sum coefficient x signal in f64) with TextFieldData::bm25 re-seeking its own cursors
 *         core/src/collector/top_docs.rs:404-490, core/src/ranking/initial.rs:79-93,
 *         core/src/ranking/computer/mod.rs:109-124, core/src/ranking/bm25.rs:97-102,136-150
 * The posting bytes are consumed exactly as tantivy writes them (128-doc BitPacker4x blocks, strict
 * deltas, tf-1, VInt tail, skip entries: tantivy/src/postings/{serializer.rs:365-462,skip.rs:186-238}).
 *
 * The GPU scores exhaustively (every posting of every query term) and returns the exact top-k under the
 * reference's total order (score descending, then doc ascending; tantivy/src/collector/top_collector.rs:50-66).
 * Pruning in the reference (Block-WAND, TopNComputer threshold) only drops documents that cannot enter the
 * top-k, so results are identical.  f32/f64 expressions are evaluated in the reference's operation order
 * without FMA contraction; see DESIGN.md for the one documented deviation (the association of the f32 sum
 * in tantivy OR queries with >= 3 terms, which in the reference depends on the pruning history).
 */
#ifndef STRACT_B200_BM25_H
#define STRACT_B200_BM25_H
#include "stract_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct sb200_segment sb200_segment;
typedef struct sb200_signals sb200_signals;

/* TermInfo{doc_freq, postings_range} of one term, tantivy/src/postings/term_info.rs:9-14 */
typedef struct { uint64_t postings_off; uint64_t postings_len; uint32_t doc_freq; uint32_t _pad; } sb200_term_info;

#define SB200_RECORD_BASIC 0            /* IndexRecordOption::Basic: 5-byte skip entries, no tf */
#define SB200_RECORD_FREQS 1            /* WithFreqs: 8-byte skip entries */
#define SB200_RECORD_FREQS_POSITIONS 2  /* WithFreqsAndPositions: 12-byte skip entries */

/* Opens one field of one segment (InvertedIndexReader + FieldNormReader, tantivy/src/index/
 * inverted_index_reader.rs:66-68, tantivy/src/fieldnorm/reader.rs:128-136): copies the postings file and the
 * 1-byte-per-doc fieldnorm ids into HBM and builds a per-block directory (last doc, byte offset, bit widths)
 * from the skip lists so blocks are randomly addressable on the device.  Terms are addressed by their ordinal
 * in `terms` afterwards. */
SB200_API int sb200_segment_create(const uint8_t* postings_file, uint64_t postings_len, const sb200_term_info* terms,
                                   uint32_t n_terms, const uint8_t* fieldnorm_ids, uint32_t max_doc,
                                   int record_option, int device, sb200_segment** out);
SB200_API void sb200_segment_destroy(sb200_segment* seg);

/* The "term ordinal -> TermInfo" half of the term dictionary (SURVEY 8(f) rank 2): decodes a whole tantivy TermInfoStore
 * (tantivy/src/termdict/fst_termdict/term_info_store.rs: 256-term blocks, a 47-byte TermInfoBlockMeta each, bit-packed
 * offsets) on the device, one thread per ordinal, into the array sb200_segment_create takes.  `store` may be host or
 * device memory, `infos` receives min(cap, n) entries, *n_terms the number of terms.  (The FST that maps term bytes to an
 * ordinal is an external crate that is not part of the reference tree; callers address terms by ordinal.) */
SB200_API int sb200_term_info_store_decode(const uint8_t* store, uint64_t len, int device, sb200_term_info* infos, uint64_t cap,
                                           uint64_t* n_terms);

typedef struct { uint64_t n_terms, n_blocks, n_postings, hbm_bytes; uint32_t max_doc; uint32_t _pad; double stage_ms; } sb200_segment_info;
SB200_API int sb200_segment_get_info(const sb200_segment* seg, sb200_segment_info* info);

/* Row-major table of per-document numeric signal scores in HBM ([max_doc][n_cols] f64): what the numeric
 * CoreSignals read per candidate (core/src/ranking/signals/core/non_text.rs).  Column j holds the signal's
 * *score* (the host applies value->score transforms such as score_rank once at open time). */
SB200_API int sb200_signals_create(const double* const* columns, uint32_t n_cols, uint32_t max_doc, int device, sb200_signals** out);
/* The same table built from the RAW fast-field columns: the library applies the numeric CoreSignals' value -> score
 * transforms (core/src/ranking/signals/core/non_text.rs) on the device, one pass per column at open time.
 *   kind                   reference                                            raw column
 *   SB200_NUM_IDENTITY     HostCentrality, PageCentrality (:117-155, :203-241)  f64
 *   SB200_NUM_RANK         score_rank (:50-59): HostCentralityRank, PageCentralityRank   u64  (evaluated on the host: libm ln)
 *   SB200_NUM_BOOL         IsHomepage (:289-332)                                bool8
 *   SB200_NUM_BOOL_NOT     HasAds: score = !likely_has_ads (:730-771)           bool8
 *   SB200_NUM_INVERSE      score_trackers / score_digits / score_slashes (:61-74): TrackerScore, UrlDigits, UrlSlashes   u64
 *   SB200_NUM_FETCH_TIME   FetchTimeMs over fetch_time_ms_cache (1000 entries, computer/mod.rs:257-259)                  u64
 *   SB200_NUM_UPDATE_TIME  UpdateTimestamp: score_timestamp (:25-42) over update_time_cache; p0 = current_timestamp      u64
 *   SB200_NUM_LINK_DENSITY score_link_density (:76-83)                          f64
 *   SB200_NUM_REGION       score_region (:85-101): lut[region id] = RegionCount::score (count / total, webpage/region.rs:219-227),
 *                          p1 != 0: a region other than All is selected, p0 = its id (+50); lut NULL = no RegionCount: all 0     u64 */
#define SB200_NUM_IDENTITY 0u
#define SB200_NUM_RANK 1u
#define SB200_NUM_BOOL 2u
#define SB200_NUM_BOOL_NOT 3u
#define SB200_NUM_INVERSE 4u
#define SB200_NUM_FETCH_TIME 5u
#define SB200_NUM_UPDATE_TIME 6u
#define SB200_NUM_LINK_DENSITY 7u
#define SB200_NUM_REGION 8u
#define SB200_NUM_U64 0u
#define SB200_NUM_F64 1u
#define SB200_NUM_BOOL8 2u
typedef struct {
  uint32_t kind, dtype;      /* SB200_NUM_* transform, SB200_NUM_U64 / F64 / BOOL8 element type of `raw` */
  const void* raw;           /* [max_doc], host or device */
  double p0, p1;
  const double* lut; uint32_t lut_len, _pad;
} sb200_numeric_column;
SB200_API int sb200_signals_create_raw(const sb200_numeric_column* cols, uint32_t n_cols, uint32_t max_doc, int device, sb200_signals** out);
/* rows [first_doc, first_doc + n_docs) of the table, row-major [n_docs][n_cols] (inspection / tests) */
SB200_API int sb200_signals_read(const sb200_signals* s, uint32_t first_doc, uint32_t n_docs, double* rows_out);
SB200_API void sb200_signals_destroy(sb200_signals* s);

#define SB200_MODE_AND 0     /* all clauses Occur::Must  -> Intersection, score = left + right + sum(others) */
#define SB200_MODE_OR 1      /* all clauses Occur::Should -> union, score = f32 sum over matching terms in query order */
#define SB200_MODE_OR_WAND 2 /* the same union with tantivy's Block-Max WAND replayed step by step (block_wand.rs:148-214): the f32
                               sum of a document's term scores then has the association the reference's pruning history gives it,
                               so scores and doc order match the reference bit for bit for ANY number of terms.  10-100x slower
                               than SB200_MODE_OR, whose sums are in query order (identical for <= 2 terms). */
#define SB200_NO_TERM 0xFFFFFFFFu  /* padding for queries shorter than the batch arity */
#define SB200_MAX_QUERY_TERMS 8
#define SB200_MAX_K 4096

/* A batch of same-arity queries over one field.  Weights come from the host exactly as the reference computes
 * them: `weight[q][t]` = Bm25Weight.weight (idf*(1+K1), tantivy/src/query/bm25.rs:161-162) for path A or the
 * Stract idf (core/src/ranking/bm25.rs:124-134) for path B; `tf_cache256` = the field's 256-entry
 * K1*(1-B+B*fieldnorm/avg) table (bm25.rs:58-68), shared by every term of the field. */
typedef struct {
  uint32_t n_queries, n_terms;
  const uint32_t* term_ords;   /* [n_queries*n_terms], SB200_NO_TERM to pad */
  const float* weights;        /* [n_queries*n_terms] */
  const float* tf_cache256;    /* [256] */
  int mode;                    /* SB200_MODE_AND / SB200_MODE_OR */
  uint32_t k;                  /* TopDocs::with_limit(k) */
} sb200_bm25_batch;

/* ms: device time of the whole call on the handle's stream (query H2D + kernel + result D2H);
 * kernel_ms: the top-k kernels alone, from the first launch to the end of the last (the doc-range merge included),
 * CUDA events around them. */
typedef struct { uint64_t postings_scored; uint64_t docs_scored; uint64_t blocks_decoded; float ms; float kernel_ms; } sb200_bm25_stats;

/* Path A.  Outputs are host (or device) arrays: docs/scores [n_queries*k] in rank order (score desc, doc asc),
 * n_out[q] <= k entries valid per query. */
SB200_API int sb200_bm25_topk_batch(sb200_segment* seg, const sb200_bm25_batch* batch, uint32_t* docs, float* scores,
                                    uint32_t* n_out, sb200_bm25_stats* stats);
/* single query convenience (a batch of one) */
SB200_API int sb200_bm25_topk(sb200_segment* seg, const uint32_t* term_ords, const float* weights, uint32_t n_terms,
                              const float* tf_cache256, int mode, uint32_t k, uint32_t* docs, float* scores, uint32_t* n_out);

/* Path B.  Candidates = union of the query terms' postings (MainCollector does not require scoring, the docset
 * is the Should-union), per candidate
 *   total = coeff_text * (bm25 as f64) + sum_j coeffs[j] * signals[doc][j]        (f64, that order)
 *   bm25  = f32 sum over the query terms in query order of idf*((tf*(k1+1))/(tf+cache[fieldnorm_id])), tf=0 -> 0
 * top-k by (total desc, doc asc).  max_docs > 0 stops after that many candidates in ascending doc order
 * (ShortCircuitQuery, tantivy/src/query/shortcircuit.rs:100-133). */
typedef struct {
  sb200_bm25_batch q;          /* mode ignored (always the union); weights = Stract idf */
  float k1;                    /* Bm25Constants.k1 of the field (1.2) */
  double coeff_text;           /* coefficient of the field's BM25 signal */
  const sb200_signals* signals;/* nullable */
  const double* coeffs;        /* [signals.n_cols] */
  uint32_t max_docs; uint32_t _pad;
} sb200_signal_batch;
SB200_API int sb200_signal_topk_batch(sb200_segment* seg, const sb200_signal_batch* batch, uint32_t* docs, double* totals,
                                      uint32_t* n_out, sb200_bm25_stats* stats);

/* Path B over SEVERAL text fields of one segment (SURVEY 8(f) rank 3): the recall-stage signal set of
 * SignalComputeOrder::compute (core/src/ranking/computer/order.rs:17-135) evaluated per candidate exactly as
 * InitialSegmentScoreTweaker::score sums it (core/src/ranking/initial.rs:79-93):
 *     total = sum over the ops, in the order given, of coeff * score            (f64)
 * A field is one sb200_segment (the same tantivy segment opened per field: equal max_doc).  A query gives every field
 * its terms as SLOTS in query order -- slot_field[q][x] = field index (0xFF pads), slot_term = the term's ordinal in that
 * field's segment or SB200_NO_TERM when the segment does not hold it (SegmentPostings::empty(): the slot still counts in
 * num_query_terms), slot_idf = MultiBm25Weight's idf (core/src/ranking/bm25.rs:52-92), slot_idf_f = MultiBm25FWeight's
 * (doc_freq of the AllBody field, core/src/ranking/bm25f.rs:40-45,88-131).  Op kinds (computer/mod.rs:66-163):
 *   SB200_OP_BM25      TextFieldData::bm25 of `field`      f32 sum over its slots of idf*((tf*(k1+1))/(tf+cache[id])), tf=0 -> 0
 *   SB200_OP_BM25F     Bm25F: f64 sum over the fields (in field order) of TextFieldData::bm25f -- the same saturation
 *                      with slot_idf_f and tf scaled by the field's bm25f_coefficient as f32 (bm25f.rs:167-180)
 *   SB200_OP_COVERAGE  matching slots / num_query_terms of `field` (f64)
 *   SB200_OP_IDF_SUM   f32 sum of slot_idf over the matching slots of `field`
 *   SB200_OP_NUMERIC   column `col` of the signal table
 * chain != 0 marks the members of an n-gram group in the reference's order (largest n first; 1 = first member):
 * score *= 0.4^hits and hits += (score > 0) (NGRAM_DAMPENING, computer/order.rs:95-135).
 * Optic rule boosts (SignalComputer::boosts, computer/mod.rs:471-497): a rule whose docset is one posting list is a slot
 * with slot_field = field | 0x80 and its boost in slot_boost (negative = downrank); rule slots are probed for the documents
 * being scored and never produce candidates; total *= (downrank > boost ? 1/(1 + downrank - boost) : boost - downrank + 1)
 * with the f64 sums taken in slot order.  slot_boost may be NULL when no slot is a rule.
 * Candidates are the union of the TEXT slots' postings; top-k by (total desc, doc asc).  Limits: <= 6 fields, <= 16 slots
 * per query, <= 32 ops. */
#define SB200_OP_BM25 0u
#define SB200_OP_BM25F 1u
#define SB200_OP_COVERAGE 2u
#define SB200_OP_IDF_SUM 3u
#define SB200_OP_NUMERIC 4u
typedef struct { sb200_segment* seg; const float* tf_cache256; float k1; float bm25f_coefficient; } sb200_signal_field;
typedef struct { uint32_t kind, field, chain, col; double coeff; } sb200_signal_op;
typedef struct {
  uint32_t n_queries, n_slots;        /* slots per query (row width of the four arrays below) */
  const uint8_t* slot_field;          /* [n_queries*n_slots] */
  const uint32_t* slot_term;          /* [n_queries*n_slots] */
  const float* slot_idf;              /* [n_queries*n_slots] */
  const float* slot_idf_f;            /* [n_queries*n_slots] */
  uint32_t n_fields, n_ops;
  const sb200_signal_field* fields;   /* [n_fields], in TextFieldEnum order */
  const sb200_signal_op* ops;         /* [n_ops], in SignalComputeOrder order */
  const sb200_signals* signals;       /* nullable unless an op is SB200_OP_NUMERIC */
  uint32_t k, _pad;
  const double* slot_boost;           /* [n_queries*n_slots], read for rule slots only; nullable */
} sb200_multi_signal_batch;
SB200_API int sb200_multi_signal_topk_batch(const sb200_multi_signal_batch* batch, uint32_t* docs, double* totals, uint32_t* n_out,
                                            sb200_bm25_stats* stats);

/* Host-side writer of tantivy-format posting lists (PostingsSerializer for IndexRecordOption::WithFreqs,
 * tantivy/src/postings/serializer.rs:343-462), used to build synthetic / test segments.  Terms are given
 * CSR-style: term t owns docs[term_off[t]..term_off[t+1]) (ascending) and the matching tfs (>= 1).
 * Call with out == NULL to get the byte size. */
SB200_API int sb200_postings_encode(const uint32_t* docs, const uint32_t* tfs, const uint64_t* term_off, uint32_t n_terms,
                                    const uint8_t* fieldnorm_ids, uint32_t max_doc, float avg_fieldnorm, uint8_t* out,
                                    uint64_t out_cap, uint64_t* out_len, sb200_term_info* infos, int threads);
/* The same writer with the record option spelled out: 1 = WithFreqs (8-byte skip entries), 2 = WithFreqsAndPositions,
 * what Stract's position-bearing text fields use (core/src/schema/text_field.rs:124-130): 12-byte skip entries that carry
 * the block's term-frequency sum (tantivy/src/postings/skip.rs:52-76,217-232); the positions themselves are another file. */
SB200_API int sb200_postings_encode_ex(const uint32_t* docs, const uint32_t* tfs, const uint64_t* term_off, uint32_t n_terms,
                                       const uint8_t* fieldnorm_ids, uint32_t max_doc, float avg_fieldnorm, int record_option,
                                       uint8_t* out, uint64_t out_cap, uint64_t* out_len, sb200_term_info* infos, int threads);
/* ---- positions and phrase queries (tantivy path A for PhraseQuery) ------------------------------------------------------
 * Host-side PositionSerializer (tantivy/src/positions/serializer.rs:47-87) for synthetic / test segments.  Input is CSR by
 * term and posting: term t owns postings [term_off[t], term_off[t+1]); posting p owns tfs[p] absolute, ascending positions,
 * concatenated in posting order in `positions`.  Each posting's positions become deltas (the first one against 0, u32
 * arithmetic like the recorder), 128 deltas are one compress_block_unsorted block, the rest of a term is a VInt tail.  The
 * output is the field's `.pos` bytes and every term's byte range.  Call with out == NULL to get the byte size. */
SB200_API int sb200_positions_encode(const uint32_t* positions, const uint32_t* tfs, const uint64_t* term_off, uint32_t n_terms,
                                     uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* positions_off,
                                     uint64_t* positions_len);
/* Attaches a field's positions file (PositionReader, tantivy/src/positions/reader.rs) to a segment opened with
 * SB200_RECORD_FREQS_POSITIONS: copies the bytes into HBM and builds, on the device, the byte offset of every bit-packed
 * positions block and the position offset of every posting block (the prefix of the skip entries' term-frequency sums,
 * tantivy/src/postings/skip.rs:219,261-266).  positions_off / positions_len [n_terms] are the terms' byte ranges in the file
 * (TermInfo.positions_range).  A segment with another record option is rejected with SB200_EINVAL (PhraseQuery's
 * SchemaError, phrase_query.rs:106-118); ranges outside the file, malformed VInt headers or tails and bit widths > 32 with
 * SB200_EFORMAT.  Attaching again replaces the previous positions. */
SB200_API int sb200_segment_attach_positions(sb200_segment* seg, const uint8_t* positions_file, uint64_t len,
                                             const uint64_t* positions_off, const uint64_t* positions_len);
/* PositionReader::read on the device decoder: the n position DELTAS [offset, offset + n) of term `term` into `out` (host or
 * device).  SB200_ERANGE when the term has fewer positions. */
SB200_API int sb200_positions_read(sb200_segment* seg, uint32_t term, uint64_t offset, uint32_t n, uint32_t* out);
/* TermInfo.positions_range of every ordinal of a TermInfoStore (term_info_store.rs:63-91), next to
 * sb200_term_info_store_decode: positions_off / positions_len receive min(cap, n) entries, *n_terms the number of terms. */
SB200_API int sb200_term_info_store_decode_positions(const uint8_t* store, uint64_t len, int device, uint64_t* positions_off,
                                                     uint64_t* positions_len, uint64_t cap, uint64_t* n_terms);

#define SB200_ABSENT_TERM 0xFFFFFFFEu  /* a phrase term the segment does not hold: the phrase matches nothing (phrase_weight.rs:53-61) */
/* A batch of phrase queries over one field (PhraseWeight -> PhraseScorer -> TopNComputer).  Row q holds the phrase's terms
 * in offset order (PhraseQuery::new_with_offset_and_slop sorts them stably by offset), then SB200_NO_TERM padding; a row
 * has 2..SB200_MAX_QUERY_TERMS terms.  Duplicate terms are separate cursors.  The library intersects them in tantivy's
 * Intersection order (stable sort by doc_freq) and verifies every candidate's positions:
 *   scoring != 0  count = PhraseScorer::compute_phrase_count, match = count > 0,
 *                 score = weight[q] * (count / (count + tf_cache256[fieldnorm_id]))   (f32, bm25.rs:182-196)
 *   scoring == 0  match = PhraseScorer::phrase_exists, score = 1.0                   (EnableScoring::Disabled)
 * top-k by (score desc, doc asc). */
typedef struct {
  uint32_t n_queries, n_terms;  /* n_terms = row width */
  const uint32_t* term_ords;    /* [n_queries*n_terms] */
  const uint32_t* offsets;      /* [n_queries*n_terms] position offset of each term; NULL = 0, 1, 2, ... */
  const uint32_t* slop;         /* [n_queries]; NULL = 0 */
  const float* weights;         /* [n_queries] Bm25Weight::for_terms(...).weight; read when scoring != 0 */
  const float* tf_cache256;     /* [256]; read when scoring != 0 */
  int scoring;
  uint32_t k;
} sb200_phrase_batch;
/* candidates: documents holding every term; matches: candidates whose positions match; positions_decoded / position_bytes:
 * position deltas decoded and bytes of the position blocks and tails they come from; ms / kernel_ms as sb200_bm25_stats. */
typedef struct { uint64_t candidates, matches, positions_decoded, position_bytes; float ms, kernel_ms; } sb200_phrase_stats;
SB200_API int sb200_phrase_topk_batch(sb200_segment* seg, const sb200_phrase_batch* batch, uint32_t* docs, float* scores,
                                      uint32_t* n_out, sb200_phrase_stats* stats);

/* ---- optic pattern rules as device docsets (core/src/query/pattern_query/, core/src/query/optic.rs) ----------------------
 * A docset is a bitmap of ceil(max_doc / 32) u32 words in HBM (12.5 MB at 100 M docs), bit d = document d, on the device of
 * the segment it was built from.  Optic rules only ever ask "is doc d in it?", so AND / OR of bitmaps is their exact
 * composition (a rule = OR over its Matches blocks of the AND of the block's matchings, optic.rs:104-169). */
typedef struct sb200_docset sb200_docset;
#define SB200_PART_PAD 0u       /* padding behind a pattern's parts */
#define SB200_PART_TERM 1u      /* PatternPart::Raw after tokenisation: one part per token, its ordinal in term_ords */
#define SB200_PART_WILDCARD 2u  /* PatternPart::Wildcard */
#define SB200_PART_ANCHOR 3u    /* PatternPart::Anchor */
/* A batch of PatternQuerys over one field, parts as PatternQuery::new leaves them (every raw part tokenised into TERM parts).
 * The library chooses PatternWeight::pattern_scorer's branch (weight.rs:121-226):
 *   no parts -> empty;  no TERM and a WILDCARD -> every document;  no TERM, anchors only -> the documents whose token count is 0;
 *   an SB200_ABSENT_TERM -> empty;  one TERM and nothing else -> its postings;
 *   otherwise NormalPatternScorer (scorer.rs:203-339): the AND of the terms, then per document left = positions of term 0 and,
 *   for every later TERM, left = { r in positions(term) : some l in left with r - slop <= l <= r } (saturating; slop 1, or
 *   u32::MAX after a WILDCARD); the document matches when the last left is non-empty, an ANCHOR at index 0 holds (the first
 *   position of term 0 is 0) and an ANCHOR at the last index holds (the last position of the last term equals
 *   (token count - 1) as u32).  Anchors elsewhere are ignored.
 * Row p has parts[p * n_parts ..] (SB200_PART_PAD behind) and the ordinals of its TERM parts in order in
 * term_ords[p * n_terms ..]; at most SB200_MAX_QUERY_TERMS terms per pattern (SB200_ERANGE above).  Patterns with a TERM and
 * another part need positions (sb200_segment_attach_positions); anchored and empty-field patterns need the token-count
 * column (sb200_segment_attach_token_counts), else SB200_EINVAL.  out[p] receives a new docset per row. */
typedef struct {
  uint32_t n_patterns, n_parts;  /* n_parts = row width of parts */
  const uint8_t* parts;          /* [n_patterns * n_parts] SB200_PART_* */
  uint32_t n_terms, _pad;        /* row width of term_ords */
  const uint32_t* term_ords;     /* [n_patterns * n_terms] ordinals or SB200_ABSENT_TERM; entries past the row's TERM count are ignored */
} sb200_pattern_batch;
/* candidates: documents holding every term of a positional pattern; matches: those that matched; positions_decoded /
 * position_bytes as sb200_phrase_stats; ms: the whole call, kernel_ms: the launches (CUDA events). */
typedef struct { uint64_t candidates, matches, positions_decoded, position_bytes; float ms, kernel_ms; } sb200_pattern_stats;
SB200_API int sb200_pattern_docsets(sb200_segment* seg, const sb200_pattern_batch* batch, sb200_docset** out, sb200_pattern_stats* stats);
/* The field's token-count fast field (NumTitleTokens, NumCleanBodyTokens, ...; weight.rs:129-160), one u64 per document, a
 * missing value passed as 0 (EmptyFieldScorer's unwrap_or_default; NormalPatternScorer unwraps it, so an anchored pattern over
 * a document without a value is outside the reference's domain).  Host or device memory; attaching again replaces it. */
SB200_API int sb200_segment_attach_token_counts(sb200_segment* seg, const uint64_t* counts, uint32_t max_doc);
/* the posting list of one term as a docset (FastSiteDomainPatternWeight: `|raw|` on Site / Domain reads the concatenated raw
 * text in the no-tokenizer field, pattern_query/mod.rs:61-92,166-175; also any rule whose docset is one posting list).
 * SB200_ABSENT_TERM gives the empty docset. */
SB200_API int sb200_docset_from_postings(sb200_segment* seg, uint32_t term, sb200_docset** out);
#define SB200_DOCSET_AND 0
#define SB200_DOCSET_OR 1
/* AND / OR of n >= 1 docsets with the same max_doc and device (fields of one tantivy segment) into a new docset */
SB200_API int sb200_docset_combine(int op, const sb200_docset* const* inputs, uint32_t n, sb200_docset** out);
SB200_API int sb200_docset_count(const sb200_docset* ds, uint64_t* count);
/* the first min(cap, total) documents in ascending order into docs (host or device), the number of documents into *total */
SB200_API int sb200_docset_read(const sb200_docset* ds, uint32_t* docs, uint64_t cap, uint64_t* total);
SB200_API int sb200_docset_info(const sb200_docset* ds, uint32_t* max_doc, int* device);
SB200_API void sb200_docset_destroy(sb200_docset* ds);

/* The multi-field recall stage (sb200_multi_signal_topk_batch) with optic rules given as docsets.  Per query q:
 *   rule_docset[q][r] (r < n_rules[q] <= SB200_MAX_OPTIC_RULES): an index into `docsets`, rule_boost[q][r] its f64 boost
 *     (negative = downrank) -- SignalComputer's Boost / Downrank rules with b != 0 in rule order (computer/mod.rs:267-277).
 *     A document in the rule's docset adds |b| to downrank or b to boost, in rule order; the total is multiplied by the
 *     factor of sb200_multi_signal_topk_batch.
 *   exclude[q]: a docset index or SB200_NO_DOCSET: the OR of the Discard rules and blocked hosts (MustNot).
 *   require[q]: a docset index or SB200_NO_DOCSET: with DiscardNonMatching, the AND over optics of the OR of their non-Discard
 *     rules (Must).
 * A candidate in exclude or outside require is dropped before it is scored (query/mod.rs:129-137, optic.rs:50-89).  Rule
 * slots (field | 0x80) and docset rules in one query are SB200_EINVAL: their relative order would be undefined.  Every docset
 * must have the segment's max_doc and device.  An optic with no rules and no filters gives the bits of
 * sb200_multi_signal_topk_batch. */
#define SB200_MAX_OPTIC_RULES 64
#define SB200_NO_DOCSET 0xFFFFFFFFu
typedef struct {
  uint32_t n_docsets, max_rules;        /* max_rules = row width of rule_docset / rule_boost */
  const sb200_docset* const* docsets;   /* [n_docsets] */
  const uint32_t* n_rules;              /* [n_queries]; NULL = no rules */
  const uint32_t* rule_docset;          /* [n_queries * max_rules] */
  const double* rule_boost;             /* [n_queries * max_rules] */
  const uint32_t* exclude;              /* [n_queries]; NULL = none */
  const uint32_t* require;              /* [n_queries]; NULL = none */
} sb200_optic_batch;
SB200_API int sb200_multi_signal_topk_batch_optic(const sb200_multi_signal_batch* batch, const sb200_optic_batch* optic, uint32_t* docs,
                                                  double* totals, uint32_t* n_out, sb200_bm25_stats* stats);

/* ---- the recall docset of Stract's query plan (core/src/query/plan/, Query::parse in core/src/query/mod.rs:106-122) ----------
 * A query's plan, compiled to a tantivy BooleanQuery and evaluated with scoring disabled, is a post-order program of nodes:
 *   SB200_PLAN_TERM    segment, arg = term ordinal or SB200_ABSENT_TERM (an empty TermScorer): the term's postings
 *   SB200_PLAN_PHRASE  segment, arg = a row of the phrase table (terms and offsets as in sb200_phrase_batch, slop per row):
 *                      PhraseScorer::phrase_exists (scoring is disabled); a row with an SB200_ABSENT_TERM matches nothing.  The
 *                      segment needs positions (SB200_RECORD_FREQS_POSITIONS and sb200_segment_attach_positions).
 *   SB200_PLAN_EMPTY   BooleanQuery::new(vec![]): matches nothing
 *   SB200_PLAN_BOOL    the n_children nodes before it (each a subtree) are its clauses, with their `occur`; BooleanWeight
 *                      (boolean_weight.rs:107-180): no clauses -> empty; one MustNot clause alone -> empty; one other clause ->
 *                      that clause; otherwise the Must intersection (Should clauses are ignored when a Must exists) or else the
 *                      Should union, minus the MustNot union; neither Must nor Should -> empty.
 * `occur` is the node's occur in its parent (SB200_PLAN_MUST / SHOULD / MUST_NOT); the root's is ignored.  Query q owns nodes
 * [node_off[q], node_off[q + 1]), at most SB200_PLAN_MAX_NODES, and the program must leave exactly one value.  Plan segments are
 * their own array: leaves span fields that are not signal fields (UrlForSiteOperator, Links, compound fields).  Every segment
 * must have the same max_doc and device (fields of one tantivy segment).  Malformed programs, bad indices and mismatched
 * segments are SB200_EINVAL. */
#define SB200_PLAN_TERM 0u
#define SB200_PLAN_PHRASE 1u
#define SB200_PLAN_EMPTY 2u
#define SB200_PLAN_BOOL 3u
#define SB200_PLAN_MUST 0u
#define SB200_PLAN_SHOULD 1u
#define SB200_PLAN_MUST_NOT 2u
#define SB200_PLAN_MAX_NODES 256
typedef struct { uint8_t kind, occur; uint16_t n_children; uint32_t segment; uint32_t arg; uint32_t _pad; } sb200_plan_node;
typedef struct {
  uint32_t n_queries, n_segments;
  sb200_segment* const* segments;   /* [n_segments] */
  const uint32_t* node_off;         /* [n_queries + 1] */
  const sb200_plan_node* nodes;     /* [node_off[n_queries]] */
  uint32_t n_phrases, phrase_terms; /* rows of the phrase table, row width (2..SB200_MAX_QUERY_TERMS, SB200_NO_TERM pads a row's end) */
  const uint32_t* phrase_ords;      /* [n_phrases * phrase_terms] ordinals or SB200_ABSENT_TERM; NULL when no node is a PHRASE */
  const uint32_t* phrase_offsets;   /* [n_phrases * phrase_terms] position offset of each term; NULL = 0, 1, 2, ... */
  const uint32_t* phrase_slop;      /* [n_phrases]; NULL = 0 */
} sb200_recall_plan_batch;
/* cover: candidates decoded (a superset of each query's docset, see DESIGN.md), docs: documents in the docsets, groups: query
 * groups the candidate budget split the batch into; ms: the whole call, kernel_ms: the launches (CUDA events). */
typedef struct { uint64_t cover, docs; uint32_t groups, _pad; float ms, kernel_ms; } sb200_plan_stats;
/* Every query's plan docset: counts[q] documents, the first min(cap, counts[q]) of them ascending in docs[q * cap ..].
 * docs may be NULL when cap == 0.  counts and docs may be host or device memory. */
SB200_API int sb200_recall_plan_docs(const sb200_recall_plan_batch* plan, uint64_t* counts, uint32_t* docs, uint64_t cap,
                                     sb200_plan_stats* stats);
/* The multi-field recall stage (sb200_multi_signal_topk_batch, same slots, ops and outputs) over exactly each query's plan
 * docset, after the optic filters of sb200_multi_signal_topk_batch_optic (optic nullable): BooleanQuery[(Must, plan), optic
 * clauses...] (query/mod.rs:133-137).  A document that no slot holds is scored with every text signal 0.  The plan batch
 * must have as many queries as the signal batch and the segments the signal fields' max_doc and device.
 * stats->docs_scored counts the documents scored, kernel_ms covers both stages. */
SB200_API int sb200_multi_signal_topk_batch_plan(const sb200_multi_signal_batch* batch, const sb200_recall_plan_batch* plan,
                                                 const sb200_optic_batch* optic, uint32_t* docs, double* totals, uint32_t* n_out,
                                                 sb200_bm25_stats* stats);

/* ---- the recall webpages of Stract's searcher (retrieve_ranking_websites, core/src/inverted_index/search.rs:110-192) ----------
 * For a GIVEN list of documents per query, what LocalRecallRankingWebpage::new (core/src/ranking/pipeline/stages/recall.rs:167-220)
 * takes from the SignalComputer, evaluated with the slots, ops and optic rules of the top-k entry points (same batch, same optic
 * batch; optic nullable):
 *   values / scores [n_queries][n_docs_max][n_ops]  op o's SignalCalculation { value, score } (compute_signals, signals/mod.rs:376-388):
 *       BM25, BM25F, COVERAGE, IDF_SUM: value = the op's score before n-gram dampening, score = after it (computer/order.rs:113-136);
 *       NUMERIC: score = the signal table's column; value is NOT written -- a numeric CoreSignal's value is its raw fast-field
 *       value as f64 (signals/core/non_text.rs), which the caller holds.
 *     sum over o (in op order) of coeff_o * score_o, times boost, is bit for bit the total the top-k entry points give the document.
 *   boosts [n_queries][n_docs_max]  SignalComputer::boosts (computer/mod.rs:471-497) over the rule slots and the docset rules; 1.0
 *       without rules.  The optic exclude / require filters are NOT applied: the caller chose the documents.
 *   min_slop [n_queries][n_docs_max][2]  per distance field (dist_field[0] = Title, [1] = CleanBody) min_slop of term_distance.rs:23-54
 *       over the field's TEXT slots in slot order (rule slots are not postings of the field; duplicate terms are separate slots),
 *       positions absolute (positions_with_offset(0)): the max over consecutive slot pairs of the least b - a with a in the left
 *       list and b > a in the right one.  0xFFFFFFFF (u32::MAX) when the field is not registered, has fewer than 2 slots, or a slot
 *       lacks the document (an absent term included: SegmentPostings::empty()).  MinTitleSlop / MinCleanBodySlop are then
 *       { value: v as f64, score: 1.0 / (v as f64 + 1.0) } in f64.
 * Documents may come in any order and repeat; every output follows the caller's order (search.rs restores orig_index).  docs and
 * n_docs are host memory; the four outputs host or device memory.  Entries past n_docs[q] are 0 (values: left as they were).
 * SB200_EINVAL: a doc >= max_doc, n_docs[q] > n_docs_max, a distance field index >= n_fields or both the same, a distance field
 * whose segment has no positions attached (sb200_segment_attach_positions), rule slots and docset rules in one query; the batch's
 * limits are those of sb200_multi_signal_topk_batch (k is not read).  Scratch grows with the batch; SB200_ENOMEM when it cannot. */
#define SB200_WEBPAGE_NO_FIELD 0xFFFFFFFFu
typedef struct {
  uint32_t n_queries, n_docs_max;   /* n_queries must equal the signal batch's; n_docs_max = row width of docs */
  const uint32_t* docs;             /* [n_queries * n_docs_max] */
  const uint32_t* n_docs;           /* [n_queries] */
  uint32_t dist_field[2];           /* indices into batch->fields of Title and CleanBody, SB200_WEBPAGE_NO_FIELD when not registered */
} sb200_webpage_batch;
typedef struct {
  double* values;                   /* [n_queries][n_docs_max][n_ops] */
  double* scores;                   /* [n_queries][n_docs_max][n_ops] */
  double* boosts;                   /* [n_queries][n_docs_max] */
  uint32_t* min_slop;               /* [n_queries][n_docs_max][2] */
} sb200_webpage_out;
/* docs: documents evaluated; docs_with_positions: documents with at least one distance field decided by its positions;
 * positions_decoded / position_bytes as sb200_phrase_stats; ms: the whole call, kernel_ms: the launches (CUDA events). */
typedef struct { uint64_t docs, docs_with_positions, positions_decoded, position_bytes; float ms, kernel_ms; } sb200_webpage_stats;
SB200_API int sb200_multi_signal_webpages(const sb200_multi_signal_batch* batch, const sb200_optic_batch* optic,
                                          const sb200_webpage_batch* wb, const sb200_webpage_out* out, sb200_webpage_stats* stats);

/* idf(doc_freq, doc_count) = ln(1 + (N - n + 0.5) / (n + 0.5)) in f32 (tantivy/src/query/bm25.rs:52-56,
 * core/src/ranking/bm25.rs:23-27) for an array of doc_freqs; tantivy_weight != 0 returns Bm25Weight.weight = idf * (1 + K1). */
SB200_API int sb200_bm25_idf(const uint32_t* doc_freq, uint64_t n, uint64_t doc_count, int tantivy_weight, float* out);
/* FIELD_NORMS_TABLE (tantivy/src/fieldnorm/code.rs:13-270) as the closed-form byte code it is tested against */
SB200_API uint32_t sb200_fieldnorm_id_to_value(uint8_t id);
SB200_API uint8_t sb200_fieldnorm_value_to_id(uint32_t fieldnorm);

#ifdef __cplusplus
}
#endif
#endif
