/*
 * metrics_b200 — C-ABI of the segmentation overlap-count kernel (K15), exported from the same libmetrics_b200.so as
 * include/metrics_b200.h and following its conventions: device pointers, a CUDA stream handle as the last argument,
 * 0 or a negative MB200_ERR_* code returned, message in mb200_last_error().
 *
 * Reference replaced (paths relative to src/torchmetrics/):
 *   functional/segmentation/mean_iou.py:51-61          one_hot(...).movedim(-1, 1) -> _ignore_background -> sum(p & t),
 *   functional/segmentation/dice.py:53-66                sum(t), sum(p) over every spatial axis (dice / generalized dice:
 *   functional/segmentation/generalized_dice.py:58-71    sum(p * t))
 */
#ifndef METRICS_B200_SEGMENTATION_H_
#define METRICS_B200_SEGMENTATION_H_

#include "metrics_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* bits OR-ed into err_flag by an index-format call; an out-of-range label is not counted */
#define MB200_SEG_PREDS_NEGATIVE 1u  /* a preds label < 0             */
#define MB200_SEG_PREDS_TOO_LARGE 2u /* a preds label >= num_classes  */
#define MB200_SEG_TARGET_NEGATIVE 4u /* a target label < 0            */
#define MB200_SEG_TARGET_TOO_LARGE 8u

/* input_format */
#define MB200_SEG_INDEX 0   /* preds, target: int64 labels [n, inner] (row stride inner)                                */
#define MB200_SEG_ONE_HOT 1 /* preds, target: [n, num_classes, inner], layout below, batch strides in elements         */
/* layout (one-hot only) */
#define MB200_SEG_PLANAR 0        /* class stride inner, spatial stride 1                                               */
#define MB200_SEG_CHANNELS_LAST 1 /* class stride 1, spatial stride num_classes: one_hot(x).movedim(-1, 1)              */
/* op: the elementwise product whose sum is the intersection */
#define MB200_SEG_AND 0 /* preds & target (integer dtypes) */
#define MB200_SEG_MUL 1 /* preds * target, rounded to the input dtype */

/* ------------------------------------------------------------------------------------------------
 * K15 — per-sample, per-class overlap counts.  Writes counts [3][n][C'] (intersection, pred_sum, target_sum), where
 * C' = num_classes - 1 when drop_background != 0 and num_classes > 1 (class 0 left out), else num_classes.  The planes are
 * overwritten, not accumulated into.
 *   index:   dtype tags must be MB200_I64; num_classes <= 2^31 - 1.  Counts are int64.
 *   one-hot: both tensors share one dtype tag (bool / u8 / i8 / i16 / i32 / i64 -> int64 counts of the values, summed with
 *            two's-complement wrap like torch.sum; f32 / f16 / bf16 with op MB200_SEG_MUL -> float64 sums of the values
 *            and of the products rounded to the input dtype).  The class count is num_classes.
 * Integer counts are exact and deterministic.  Float sums are deterministic: per-CTA float64 partials go to `scratch` and
 * are folded in slice order (scratch: 16-byte aligned, mb200_segmentation_scratch_bytes(...) bytes, contents irrelevant;
 * may be NULL when that size is 0).  err_flag (index format; may be NULL) receives MB200_SEG_* bits.  No host
 * synchronisation.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int64_t mb200_segmentation_scratch_bytes(int64_t n, int64_t num_classes, int64_t inner, int input_format, int layout,
                                                   int dtype, int drop_background);
MB200_API int mb200_segmentation_overlap_counts(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                                int64_t n, int64_t num_classes, int64_t inner, int input_format, int layout,
                                                int64_t preds_batch_stride, int64_t target_batch_stride, int op,
                                                int drop_background, void* counts, void* scratch, int64_t scratch_bytes,
                                                uint32_t* err_flag, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* METRICS_B200_SEGMENTATION_H_ */
