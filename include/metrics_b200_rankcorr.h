/*
 * metrics_b200 — C-ABI of the rank-correlation kernels (K17), exported from the same libmetrics_b200.so as
 * include/metrics_b200.h and following its conventions: device pointers, a CUDA stream handle as the last argument, 0 or a
 * negative MB200_ERR_* code returned, message in mb200_last_error().
 *
 * Reference replaced (paths relative to src/torchmetrics/):
 *   functional/regression/spearman.py:35-108   argsort ranking in the input dtype, one Python iteration per repeated value
 *   functional/regression/kendall.py:50-318    a Python loop over every row comparing it with all later rows (O(n^2))
 *
 * Inputs are row-major [n, d] tensors: column c of row i at index i * d + c.  Every column is ranked on its own.
 */
#ifndef METRICS_B200_RANKCORR_H_
#define METRICS_B200_RANKCORR_H_

#include "metrics_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* largest row count n: the radix sort's status words hold 30-bit counts */
#define MB200_RANKCORR_MAX_ROWS 1073741823ll

/* Kendall tau variant */
#define MB200_KENDALL_A 0
#define MB200_KENDALL_B 1
#define MB200_KENDALL_C 2

/* Kendall t-test alternative; NONE skips the p-value */
#define MB200_KENDALL_ALT_NONE 0
#define MB200_KENDALL_ALT_TWO_SIDED 1
#define MB200_KENDALL_ALT_LESS 2
#define MB200_KENDALL_ALT_GREATER 3

/* ------------------------------------------------------------------------------------------------
 * Workspace of one call: bytes for n rows of d columns, kendall = 0 (Spearman) or 1 (Kendall).  -1 when n < 0,
 * n > MB200_RANKCORR_MAX_ROWS or d < 1.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int64_t mb200_rankcorr_scratch_bytes(int64_t n, int64_t d, int kendall);

/* ------------------------------------------------------------------------------------------------
 * K17 Spearman.  preds / target: MB200_F32, F16, BF16 or F64 (tags may differ).  out[d] in out_dtype (a float tag):
 * cov(r_x, r_y) / (std(r_x) * std(r_y) + eps) with population moments of the tie-averaged ranks, clamped to [-1, 1].  NaN
 * sorts after +inf and each NaN is its own tie group; -0 equals +0.  The rank sums are exact integers, the final
 * arithmetic float64.  err_flag: receives MB200_FLAG_SPIN_TIMEOUT bits (the caller zeroes it); may be NULL.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_spearman_corrcoef(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t n,
                                      int64_t d, void* out, int out_dtype, double eps, void* scratch, int64_t scratch_bytes,
                                      uint32_t* err_flag, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K17 Kendall.  preds / target: a float tag, MB200_I32 or MB200_I64 (tags may differ).  tau[d] in tau_dtype (a float tag)
 * for `variant` (MB200_KENDALL_*), clamped to [-1, 1]; p_value[d] float32 of the asymptotic t-test for `alternative` (NULL allowed for
 * MB200_KENDALL_ALT_NONE).  Concordant / discordant pairs are counted exactly over the rows where neither value is NaN; tie
 * terms and the row count cover the whole column.  A column whose pairs are all tied has a zero t-test variance: its p-value
 * is NaN.  err_flag as for Spearman.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_kendall_rank_corrcoef(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t n,
                                          int64_t d, int variant, int alternative, void* tau, int tau_dtype, float* p_value,
                                          void* scratch, int64_t scratch_bytes, uint32_t* err_flag, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* METRICS_B200_RANKCORR_H_ */
