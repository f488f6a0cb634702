/* stract_b200_lambdamart.h -- C ABI of Stract's LambdaMART ranking model on the device (part of libstract_b200.so; conventions
 * as in stract_b200.h).
 *
 * Replaces (paths relative to crates/core/src/ in the Stract repository):
 *   LambdaMART::parse / LambdaMART::predict   ranking/models/lambdamart.rs:98-311
 *   RankingStage for Arc<LambdaMART>          ranking/pipeline/scorers/lambdamart.rs:29-42 (one batched predict per stage)
 *
 * The model text is the reference's LightGBM subset, parsed on the host exactly as the reference parses it: Rust `str::lines`,
 * the header up to the first empty line, `feature_names=` (SignalEnum names in serde's snake_case, repeated keys append), tree
 * chunks between empty lines up to the first line whose trim() is "end of trees", per tree `split_feature`, `threshold`,
 * `leaf_value`, `left_child`, `right_child` (a negative child c is leaf |c| - 1), one node slot per leaf, a slot past the end of
 * `threshold` keeps 0.0, every leaf shifted by |fold(cur < v ? cur : v)| + 1.0.  Numbers follow Rust's str::parse.
 *
 * One intended difference: the reference panics (or loops forever) when a walk reaches a node without a feature, a missing
 * child, an index out of range or a cycle.  sb200_lambdamart_load refuses such a model: every path from a root must end at a
 * leaf.  Malformed nodes that no path reaches are accepted, as in the reference.
 */
#ifndef STRACT_B200_LAMBDAMART_H
#define STRACT_B200_LAMBDAMART_H
#include "stract_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* number of SignalEnum variants (ranking/signals/mod.rs:108-155): the row width of a feature matrix */
#define SB200_SIGNAL_ENUM_COUNT 46

typedef struct sb200_lambdamart sb200_lambdamart;

/* Parses `len` bytes of model text (UTF-8, not NUL-terminated), validates it and uploads it to the current device.
 * SB200_EFORMAT: the text is not a model the reference predicts with; the message names the reference's error (NoFeatures,
 * NoEndOfTrees, ParseInt, ParseFloat, UnknownSignal, Io for invalid UTF-8) or the panic the model would cause.
 * SB200_ERANGE: a tree with 2^24 or more node slots. */
SB200_API int sb200_lambdamart_load(const char* text, uint64_t len, sb200_lambdamart** out);
SB200_API void sb200_lambdamart_destroy(sb200_lambdamart* model);

/* n_internal: internal nodes on some path from a root (the records the kernel walks); n_leaves: leaf values stored;
 * max_depth: internal nodes on the longest root-to-leaf path; device_bytes: device memory held by the handle (scratch included) */
typedef struct { uint32_t n_trees, n_features; uint64_t n_internal, n_leaves; uint32_t max_depth, _pad; uint64_t device_bytes; } sb200_lambdamart_info;
SB200_API int sb200_lambdamart_get_info(const sb200_lambdamart* model, sb200_lambdamart_info* info);
/* the SignalEnum ordinal of each header feature, in header order: min(cap, n_features) entries */
SB200_API int sb200_lambdamart_features(const sb200_lambdamart* model, uint32_t* ordinals, uint32_t cap);

/* docs: documents predicted; ms: the whole call on the handle's stream (copies included), kernel_ms: the kernel (CUDA events) */
typedef struct { uint64_t docs; float ms, kernel_ms; } sb200_lambdamart_stats;
/* LambdaMART::predict for n_docs documents: features is [n_docs][SB200_SIGNAL_ENUM_COUNT] f64 in SignalEnum order with 0.0 for
 * the signals a page lacks (the reference's EnumMap read with unwrap_or(0.0)); out[d] = the f64 sum of the trees' leaves in tree
 * order divided by the number of trees, bit for bit.  features and out may be host or device memory; stats nullable. */
SB200_API int sb200_lambdamart_predict(sb200_lambdamart* model, const double* features, uint64_t n_docs, double* out,
                                       sb200_lambdamart_stats* stats);

#ifdef __cplusplus
}
#endif
#endif
