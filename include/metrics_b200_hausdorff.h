/*
 * metrics_b200 — C-ABI of the Hausdorff-distance edge kernel (K19), exported from the same libmetrics_b200.so as
 * include/metrics_b200.h and following its conventions: device pointers, a CUDA stream handle as the last argument,
 * 0 or a negative MB200_ERR_* code returned, message in mb200_last_error().
 *
 * Reference replaced (paths relative to src/torchmetrics/):
 *   functional/segmentation/hausdorff_distance.py:94-113   one_hot of index labels, _ignore_background, a Python loop over
 *                                                          every (sample, class) pair
 *   functional/segmentation/utils.py:284-389               mask_edges (binary erosion), surface_distance and the dense
 *                                                          [pixels, edge pixels] distance_transform of the pytorch engine
 */
#ifndef METRICS_B200_HAUSDORFF_H_
#define METRICS_B200_HAUSDORFF_H_

#include "metrics_b200.h"
#include "metrics_b200_segmentation.h"

#ifdef __cplusplus
extern "C" {
#endif

/* err[0] = 4 * (first failing pair, n-major) + kind, or all ones when no pair failed */
#define MB200_HD_PREDS_NOT_BINARY 0u  /* a preds value of the pair is neither 0 nor 1 (one-hot format) */
#define MB200_HD_TARGET_NOT_BINARY 1u /* a target value of the pair is neither 0 nor 1 (one-hot format) */
#define MB200_HD_NO_EDGES 2u          /* neither mask of the pair has an edge pixel (both are empty) */

/* input_format: MB200_SEG_INDEX or MB200_SEG_ONE_HOT (include/metrics_b200_segmentation.h) */
/* metric */
#define MB200_HD_EUCLIDEAN 0
#define MB200_HD_CHESSBOARD 1
#define MB200_HD_TAXICAB 2

/* ------------------------------------------------------------------------------------------------
 * K19 — per-sample, per-class Hausdorff distance of 2-D masks.  Writes out[n][C'] (float32), C' = num_classes - 1 when
 * drop_background != 0 and num_classes > 1 (class 0 left out), else num_classes; pair q = b * C' + c'.
 *   index:   preds, target int64 labels [n, height, width] with element strides (s_n, s_h, s_w); s_c is ignored.  Class
 *            c's mask is label == c.  A label < 0 or >= num_classes ORs MB200_SEG_* bits into err[1].
 *   one-hot: preds, target [n, num_classes, height, width] of any integer dtype tag or MB200_BOOL (the two may differ),
 *            element strides (s_n, s_c, s_h, s_w).  The mask is value != 0; a value other than 0 and 1 fails the pair.
 * An edge pixel is a mask pixel with at least one of its four axis neighbours outside the mask or the image.  The directed
 * distance d(A -> B) is the maximum over edge pixels a of A of the minimum over edge pixels b of B of
 * f(|a_row - b_row|, |a_col - b_col|), f the float32 expression of the metric with spacing (s0, s1): bit k of
 * spacing_int_mask makes axis k's spacing an int64 (the value of spacing_k, integral), else spacing_k rounded to float32.
 * out = max(d(P -> T), d(T -> P)), or d(P -> T) when directed != 0; +inf when exactly one mask is empty.
 * Pairs are processed pairs_per_launch at a time in scratch (16-byte aligned, mb200_hausdorff_scratch_bytes(...) bytes,
 * contents irrelevant).  err: device uint64 [2], overwritten (err[0] above, err[1] label bits); out is undefined for the
 * update when either word reports an error.  No host synchronisation.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int64_t mb200_hausdorff_scratch_bytes(int64_t height, int64_t width, int directed, int64_t pairs_per_launch);
MB200_API int mb200_hausdorff_distance(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                       int input_format, int64_t n, int64_t num_classes, int64_t height, int64_t width,
                                       int64_t preds_s_n, int64_t preds_s_c, int64_t preds_s_h, int64_t preds_s_w,
                                       int64_t target_s_n, int64_t target_s_c, int64_t target_s_h, int64_t target_s_w,
                                       int drop_background, int metric, int spacing_int_mask, double spacing_0,
                                       double spacing_1, int directed, int64_t pairs_per_launch, float* out, void* scratch,
                                       int64_t scratch_bytes, uint64_t* err, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* METRICS_B200_HAUSDORFF_H_ */
