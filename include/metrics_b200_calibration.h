/*
 * metrics_b200 — C-ABI of the calibration-error kernels (K14), exported from the same libmetrics_b200.so as
 * include/metrics_b200.h and following its conventions: device pointers, a CUDA stream handle as the last argument,
 * 0 or a negative MB200_ERR_* code returned, message in mb200_last_error().
 *
 * Reference replaced (paths relative to src/torchmetrics/):
 *   functional/classification/calibration_error.py:239-246   _multiclass_calibration_error_update
 *       normalize_logits_if_needed(preds, "softmax") -> preds.max(dim=1) -> predictions.eq(target) -> .float()
 *       (utilities/compute.py:190-229), after the ignore_index drop of _multiclass_confusion_matrix_format
 *   functional/classification/calibration_error.py:30-61     _binning_bucketize
 *       bucketize(conf, linspace(0, 1, n_bins + 1), right=True) - 1 -> three scatter_add_ into n_bins + 1 slots
 */
#ifndef METRICS_B200_CALIBRATION_H_
#define METRICS_B200_CALIBRATION_H_

#include "metrics_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * K14a — fused top-label update, one read of preds [n, num_classes] (row-major, f32 / f16 / bf16 / f64) and of
 * target [n] (integer dtype tag).  Per row r: confidence[r] (f32) = the row maximum of
 * normalize_logits_if_needed(preds, "softmax") in the preds dtype, accuracy[r] (f32) = 1 if its first maximal index
 * (NaN maximal, first NaN wins) equals target[r], else 0.  The "are these logits?" vote is batch-global and taken over
 * the rows whose target is not `ignore_index` (has_ignore != 0); ignored rows get unspecified outputs (the caller drops
 * them).  No host synchronisation.  `scratch`: device memory of mb200_calibration_scratch_bytes(n) bytes, 16-byte
 * aligned, contents irrelevant.  `err_flag` (optional, NULL = unchecked): MB200_FLAG_TARGET_RANGE is OR-ed in when a
 * non-ignored target lies outside [0, num_classes).
 * Rows of at most 1024 f32 / f16 / bf16 scores take a speculative single pass (same bits as ATen's CUDA
 * softmax(x, 1).max(1)); wider rows and f64 take a vote pass plus a three-pass row kernel with the arithmetic of
 * mb200_curve_softmax_if_logits.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int64_t mb200_calibration_scratch_bytes(int64_t n);
MB200_API int mb200_calibration_top_label(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t n,
                                          int64_t num_classes, int has_ignore, int64_t ignore_index, float* confidence,
                                          float* accuracy, void* scratch, int64_t scratch_bytes, uint32_t* err_flag,
                                          void* stream);

/* ------------------------------------------------------------------------------------------------
 * K14b — binning.  confidences [n] (f32 / f16 / bf16 / f64), accuracies [n] (any dtype tag; each value is rounded to the
 * confidence dtype first, like the reference's `accuracies.to(confidences.dtype)`), boundaries [n_bins + 1] in the
 * confidence dtype (ascending; the caller builds them with torch.linspace).  Slot of a confidence x = (number of
 * boundaries b with !(b > x)) - 1, compared in the confidence dtype: torch.bucketize(x, boundaries, right=True) - 1.
 * NaN and x >= boundaries[n_bins] land in slot n_bins.  Writes count [n_bins + 1] (int64), sum_conf and sum_acc
 * [n_bins + 1] (float64).  Deterministic: the grid depends on n only, per-warp partials are combined in a fixed order.
 * `scratch`: device memory of mb200_calibration_bin_scratch_bytes(n, n_bins) bytes, 16-byte aligned.
 * n_bins is limited to 8191 (one warp's partial bins must fit in shared memory).
 * ------------------------------------------------------------------------------------------------ */
MB200_API int64_t mb200_calibration_bin_scratch_bytes(int64_t n, int64_t n_bins);
MB200_API int mb200_calibration_bin_sums(const void* confidences, int conf_dtype, const void* accuracies, int acc_dtype,
                                         int64_t n, const void* boundaries, int64_t n_bins, int64_t* count, double* sum_conf,
                                         double* sum_acc, void* scratch, int64_t scratch_bytes, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* METRICS_B200_CALIBRATION_H_ */
