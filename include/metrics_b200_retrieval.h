/*
 * metrics_b200 — C-ABI of the retrieval kernels (K16), exported from the same libmetrics_b200.so as include/metrics_b200.h
 * and following its conventions: device pointers, a CUDA stream handle as the last argument, 0 or a negative
 * MB200_ERR_* code returned, message in mb200_last_error().
 *
 * Reference replaced (paths relative to src/torchmetrics/):
 *   retrieval/base.py:148-183        sort by indexes, _flexible_bincount(...).cpu(), Python loop over the queries
 *   retrieval/fall_out.py:117-155    the same loop with "no negative target" emptiness
 *   functional/retrieval/*.py        the per-query topk / argsort / gather / sum of each metric
 *   retrieval/precision_recall_curve.py:205-256   the per-query curve loop and its [Q, max_k] stack
 */
#ifndef METRICS_B200_RETRIEVAL_H_
#define METRICS_B200_RETRIEVAL_H_

#include "metrics_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* metric kind of mb200_retrieval_evaluate */
#define MB200_RET_AP 0
#define MB200_RET_RR 1
#define MB200_RET_PRECISION 2
#define MB200_RET_RECALL 3
#define MB200_RET_HIT_RATE 4
#define MB200_RET_FALL_OUT 5
#define MB200_RET_R_PRECISION 6
#define MB200_RET_NDCG 7

/* largest total element count: the radix sort's status words hold 30-bit counts */
#define MB200_RET_MAX_ELEMENTS 1073741823ll

/* ------------------------------------------------------------------------------------------------
 * K16a — index range.  range[0] = min(indexes), range[1] = max(indexes) (int64 device words).  n >= 1.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_retrieval_index_range(const int64_t* indexes, int64_t n, int64_t* range, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K16b — group sort.  Orders the n records by (index ascending, score descending, position ascending): ties in score
 * keep their order in the input.  Writes
 *   keys    [n] uint64: high word = segment key, low word = ~f32_order_key(score) (NaN -> 0, -0 and +0 equal);
 *                       the segment key is index - index_min when index_max - index_min < 2^32, else the dense query rank
 *   sorted_target [n] float32: the target, converted to float32
 *   offsets [n + 1] int64: offsets[q] = first record of query q, offsets[Q] = n; entries past Q are untouched
 *   info    [2] int64: info[0] = Q (number of distinct indexes); the low word of info[1] receives MB200_FLAG_* bits
 *                       (the caller zeroes it)
 * target_dtype: MB200_I64 or MB200_F32.  scratch: mb200_retrieval_sort_scratch_bytes(n, index_bytes) bytes, 16-byte
 * aligned, where index_bytes = number of significant bytes of index_max - index_min (0..8).  Deterministic.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int64_t mb200_retrieval_sort_scratch_bytes(int64_t n, int index_bytes);
MB200_API int mb200_retrieval_sort(const int64_t* indexes, const float* preds, const void* target, int target_dtype, int64_t n,
                                   int64_t index_min, int64_t index_max, uint64_t* keys, float* sorted_target, int64_t* offsets,
                                   int64_t* info, void* scratch, int64_t scratch_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K16c — ideal order (NDCG).  ideal[n] float32 = the sorted targets of every query in descending order, queries where
 * they are in `keys` (output of K16b).  segment_bytes = significant bytes of the largest segment key (the high words).
 * scratch: mb200_retrieval_ideal_scratch_bytes(n, segment_bytes) bytes.  err_flag: may be NULL.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int64_t mb200_retrieval_ideal_scratch_bytes(int64_t n, int segment_bytes);
MB200_API int mb200_retrieval_sort_ideal(const uint64_t* keys, const float* sorted_target, int64_t n, int segment_bytes,
                                         float* ideal, void* scratch, int64_t scratch_bytes, uint32_t* err_flag, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K16d — per-query evaluation of one metric kind over the output of K16b.  value[q] float32 and empty[q] (1 when the
 * query has no positive target — for MB200_RET_FALL_OUT no negative one — else 0) for q < num_queries (int64 device
 * word).  top_k = 0 means the query length.  ideal: output of K16c for MB200_RET_NDCG, else NULL.  Warp per query up to
 * 1024 records, a CTA per longer query.  Fixed-order float64 sums: same input, same bits.  scratch:
 * mb200_retrieval_evaluate_scratch_bytes(n) bytes.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int64_t mb200_retrieval_evaluate_scratch_bytes(int64_t n);
MB200_API int mb200_retrieval_evaluate(const uint64_t* keys, const float* sorted_target, const float* ideal,
                                       const int64_t* offsets, const int64_t* num_queries, int64_t n, int kind, int64_t top_k,
                                       int adaptive_k, float* value, uint8_t* empty, void* scratch, int64_t scratch_bytes,
                                       void* stream);

/* ------------------------------------------------------------------------------------------------
 * K16e — AUROC of each query's top min(top_k, n) records (top_k = 0: all), over the output of K16b.  value[q] float32:
 * 0 when the slice has no target equal to 0 or none equal to 1; else binary_auroc of the slice with positives = targets
 * equal to 1, every score replaced by its fp32 sigmoid when a non-NaN score of the slice lies outside [0, 1], ties averaged,
 * each NaN its own group.  max_fpr < 0 or == 1: the full area; else the McClish-standardised partial area up to max_fpr
 * (which must round to a float32 below 1; 0 gives NaN).  empty[q] = 1 when the whole query has no positive target.
 * scratch: mb200_retrieval_evaluate_scratch_bytes(n) bytes.  Same scheduling and determinism as K16d.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_retrieval_auroc(const uint64_t* keys, const float* sorted_target, const int64_t* offsets,
                                    const int64_t* num_queries, int64_t n, int64_t top_k, double max_fpr, float* value,
                                    uint8_t* empty, void* scratch, int64_t scratch_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K16f — precision and recall at k = 1..max_k (max_k >= 1) of each query, over the output of K16b.  precision and recall
 * are row-major [num_queries, max_k] float32 (int64 indexing).  With cum(k) = the target sum of the top min(k, n)
 * records and P = the query's target sum: precision[q, k-1] = cum(k) / d, d = k (adaptive_k and k > n: n), recall[q, k-1]
 * = cum(k) / P, fp32 divisions.  empty[q] = 1 when P == 0; its row is zeros.  scratch:
 * mb200_retrieval_pr_curve_scratch_bytes(n) bytes.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int64_t mb200_retrieval_pr_curve_scratch_bytes(int64_t n);
MB200_API int mb200_retrieval_pr_curve(const uint64_t* keys, const float* sorted_target, const int64_t* offsets,
                                       const int64_t* num_queries, int64_t n, int64_t max_k, int adaptive_k, float* precision,
                                       float* recall, uint8_t* empty, void* scratch, int64_t scratch_bytes, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* METRICS_B200_RETRIEVAL_H_ */
