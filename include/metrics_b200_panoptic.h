/*
 * metrics_b200 — C-ABI of the panoptic-quality segment-pair counting kernel (K18), exported from the same libmetrics_b200.so
 * as include/metrics_b200.h and following its conventions: device pointers, a CUDA stream handle as the last argument,
 * 0 or a negative MB200_ERR_* code returned, message in mb200_last_error().
 *
 * Reference replaced (paths relative to src/torchmetrics/):
 *   functional/detection/_panoptic_quality_common.py:175-211   _prepocess_inputs: stuff instance ids -> 0, unknown -> void
 *   functional/detection/_panoptic_quality_common.py:312-444   per image: torch.unique(dim=0) of pred colors, target colors
 *                                                              and color pairs, then a Python loop over every pair
 */
#ifndef METRICS_B200_PANOPTIC_H_
#define METRICS_B200_PANOPTIC_H_

#include "metrics_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* bits written to err_flag by mb200_panoptic_update: MB200_PQ_UNKNOWN_PREDS, and MB200_FLAG_CAPACITY of metrics_b200.h
 * when an image has more distinct colors or color pairs than half a table (re-run larger) */
#define MB200_PQ_UNKNOWN_PREDS 1u /* a preds category is neither a thing nor a stuff (allow_unknown_preds == 0) */

/* ------------------------------------------------------------------------------------------------
 * K18 — one panoptic-quality update.  preds, target: contiguous [n, pixels, 2] (category_id, instance_id) of any integer
 * dtype tag except MB200_BOOL (the two may differ), 16-byte aligned or aligned to one (category, instance) pair.
 * categories: device int64 [2 * num_categories]: the category ids in ascending order, then the continuous id of each
 * (things 0 .. num_things - 1 in ascending id order, then stuffs).  Per image, a pixel whose category is a stuff has its
 * instance id set to 0 and one whose category is neither becomes the void color; the areas of every pred color, target
 * color and (pred, target) pair are counted in per-image hash tables, pairs of one category whose target is not void are
 * matched at IoU > 0.5 (modified != 0: stuffs at IoU > 0, counting every stuff target segment as a true positive), and
 * unmatched segments that are at most half void become false positives / negatives.  The per-image [n][K] results are
 * folded in image order and ADDED to iou_sum (float64 [K]) and true_positives, false_positives, false_negatives (int32 [K]).
 *
 * Images are processed images_per_launch at a time, each with color tables of color_capacity slots and a pair table of
 * pair_capacity slots (powers of two, 64 .. 2^31).  err_flag (required) is overwritten: MB200_PQ_UNKNOWN_PREDS, and
 * MB200_FLAG_CAPACITY when an image filled more than half a table.  With either bit set the states are left unchanged;
 * after MB200_FLAG_CAPACITY alone the caller repeats the update with capacities of at least 2 * pixels.
 * scratch: 16-byte aligned, mb200_panoptic_scratch_bytes(...) bytes, contents irrelevant.  No host synchronisation.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int64_t mb200_panoptic_scratch_bytes(int64_t n, int64_t pixels, int64_t num_categories, int64_t images_per_launch,
                                               int64_t color_capacity, int64_t pair_capacity, int preds_dtype, int target_dtype);
MB200_API int mb200_panoptic_update(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t n,
                                    int64_t pixels, const int64_t* categories, int64_t num_categories, int64_t num_things,
                                    int modified, int allow_unknown_preds, int64_t images_per_launch, int64_t color_capacity,
                                    int64_t pair_capacity, double* iou_sum, int32_t* true_positives, int32_t* false_positives,
                                    int32_t* false_negatives, void* scratch, int64_t scratch_bytes, uint32_t* err_flag,
                                    void* stream);

#ifdef __cplusplus
}
#endif

#endif /* METRICS_B200_PANOPTIC_H_ */
