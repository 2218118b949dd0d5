/*
 * metrics_b200 — C-ABI of the H100 (sm_90a) metric hot path.
 *
 * Drop-in boundary for the per-batch update()/compute() arithmetic of TorchMetrics
 * (reference = PyTorchLightning/metrics @ 1.7.0dev, paths below relative to src/torchmetrics/).
 * Every entry point is `extern "C"`, takes plain device pointers + sizes + a CUDA stream handle
 * (void* == cudaStream_t / CUstream, NULL = legacy default stream) and returns 0 on success or a
 * negative MB200_ERR_* code; `mb200_last_error()` returns a thread-local message for the last failure.
 *
 * All pointers are DEVICE pointers unless a parameter is documented as host memory.
 * Kernels are enqueued asynchronously on `stream`; no entry point synchronises the host unless stated.
 * State tensors (`confmat`, `tp` ...) are updated IN PLACE, mirroring `self.confmat += ...` in the
 * reference classes.  There is no CPU implementation behind this ABI: calling it without a CUDA device
 * fails with MB200_ERR_CUDA.
 */
#ifndef METRICS_B200_H_
#define METRICS_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MB200_ABI_VERSION 1

#if defined(__GNUC__)
#define MB200_API __attribute__((visibility("default")))
#else
#define MB200_API
#endif

/* element types accepted for preds / target buffers */
enum mb200_dtype {
    MB200_F32 = 0,
    MB200_F16 = 1,
    MB200_BF16 = 2,
    MB200_F64 = 3,
    MB200_I64 = 4,
    MB200_I32 = 5,
    MB200_I16 = 6,
    MB200_I8 = 7,
    MB200_U8 = 8,
    MB200_BOOL = 9
};

enum mb200_status {
    MB200_OK = 0,
    MB200_ERR_INVALID = -1, /* bad argument (shape, dtype, null pointer) */
    MB200_ERR_CUDA = -2,    /* CUDA runtime error, message in mb200_last_error() */
    MB200_ERR_UNSUPPORTED = -3
};

/* bits OR-ed into the optional device-side `err_flag` word by the update kernels */
#define MB200_FLAG_TARGET_RANGE 1u /* a non-ignored target label was outside [0, num_classes) */
#define MB200_FLAG_PREDS_RANGE 2u  /* an integer preds label was outside [0, num_classes)      */
#define MB200_FLAG_SPIN_TIMEOUT 4u /* internal look-back wait exceeded its bound (results invalid) */
#define MB200_FLAG_CAPACITY 8u     /* a per-image / per-class capacity of a kernel was exceeded (results invalid) */

MB200_API int mb200_abi_version(void);
MB200_API const char* mb200_last_error(void);
/* number of kernels this library has launched since load (all streams); used by bench.py `gpu_launches` */
MB200_API uint64_t mb200_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * K1 — multiclass confusion matrix update.
 * Replaces: functional/classification/confusion_matrix.py:297-328
 *           (_multiclass_confusion_matrix_format: argmax(dim=1) + flatten + ignore_index drop, then
 *            _multiclass_confusion_matrix_update: bincount(target*C + preds, C*C).reshape(C, C))
 *           + utilities/data.py:178-206 (_bincount) + classification/confusion_matrix.py:286
 *           (`self.confmat += confmat`), fused into ONE pass over the logits.
 *
 *  preds        : if preds_has_class_dim != 0: scores laid out [n_outer, num_classes, inner] contiguous
 *                 (inner = product of trailing dims, 1 for plain [N, C]); floating dtype.
 *                 else: integer (or floating holding integers is NOT accepted) labels [n_outer*inner].
 *  target       : integer labels [n_outer * inner]
 *  confmat      : int64 [num_classes, num_classes], row = target, col = prediction, updated in place
 *  ignore_index : rows whose target equals it are skipped when has_ignore_index != 0
 *  err_flag     : optional uint32 device word (may be NULL); MB200_FLAG_* bits are OR-ed in.  Rows with an
 *                 out-of-range label are skipped (the reference raises from bincount/reshape instead).
 * argmax semantics == torch.argmax: first index of the maximum, NaN is maximal (first NaN wins), -0 == +0.
 * The launch uses programmatic stream serialization and waits for the previous grid of the stream before its first
 * input load.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_multiclass_confmat_update(const void* preds, int preds_dtype, int preds_has_class_dim,
                                    const void* target, int target_dtype, int64_t n_outer,
                                    int64_t num_classes, int64_t inner, int has_ignore_index,
                                    int64_t ignore_index, int64_t* confmat, uint32_t* err_flag,
                                    void* stream);

/* ------------------------------------------------------------------------------------------------
 * K1b — multiclass stat scores update (tp / fp / tn / fn), top_k == 1, multidim_average == "global".
 * Replaces: functional/classification/stat_scores.py:328-344 (_multiclass_stat_scores_format) and
 *           :424-448 (_multiclass_stat_scores_update micro + bincount paths) + the in-place state adds of
 *           classification/stat_scores.py:69-80.  The C*C bincount is never materialised.
 *
 *  micro != 0 : tp/fp/tn/fn are int64[1]  (tp = #(p==t), fp = fn = #(p!=t), tn = C*n_valid - tp - fp - fn)
 *  micro == 0 : tp/fp/tn/fn are int64[num_classes]
 *  workspace  : int64[3*num_classes + 2] device scratch that MUST be zero on entry; the kernel leaves it
 *               zeroed again on exit (self-cleaning), so one zero-initialised buffer per metric instance
 *               can be reused forever.  It must not be shared by calls running concurrently on
 *               different streams.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_multiclass_stat_scores_update(const void* preds, int preds_dtype, int preds_has_class_dim,
                                        const void* target, int target_dtype, int64_t n_outer,
                                        int64_t num_classes, int64_t inner, int has_ignore_index,
                                        int64_t ignore_index, int micro, int64_t* tp, int64_t* fp,
                                        int64_t* tn, int64_t* fn, int64_t* workspace,
                                        uint32_t* err_flag, void* stream);

/* K1b variants.
 * top-k (functional/classification/stat_scores.py:347-368, 390-423 with top_k > 1): the effective prediction of a row is
 * its target when the target is among the k best scores, else the argmax; per-class tp/fp/tn/fn as above (micro == 0
 * layout, workspace contract identical).  preds: [n, num_classes] floating scores.
 * samplewise (multidim_average="samplewise", :390-423): per (sample, class) counts over the trailing dims;
 * counts: int64 [3][n_outer][num_classes] = tp | fp | fn planes, n_valid: int64 [n_outer]; both zero on entry;
 * tn = n_valid - tp - fp - fn is left to the caller. */
MB200_API int mb200_multiclass_stat_scores_topk_update(const void* preds, int preds_dtype, const void* target,
                                                       int target_dtype, int64_t n, int64_t num_classes, int64_t top_k,
                                                       int has_ignore_index, int64_t ignore_index, int64_t* tp,
                                                       int64_t* fp, int64_t* tn, int64_t* fn, int64_t* workspace,
                                                       uint32_t* err_flag, void* stream);
MB200_API int mb200_multiclass_stat_scores_samplewise(const void* preds, int preds_dtype, int preds_has_class_dim,
                                                      const void* target, int target_dtype, int64_t n_outer,
                                                      int64_t num_classes, int64_t inner, int has_ignore_index,
                                                      int64_t ignore_index, int64_t* counts, int64_t* n_valid,
                                                      uint32_t* err_flag, void* stream);

/* Row argmax only (the `preds.argmax(dim=1)` of the format step) — used by the samplewise / top-k host
 * paths and by tests to pin tie/NaN semantics.  out: int64 [n_outer * inner]. */
MB200_API int mb200_argmax_rows(const void* preds, int preds_dtype, int64_t n_outer, int64_t num_classes,
                      int64_t inner, int64_t* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K6 — `normalize_logits_if_needed` (utilities/compute.py:190-229, device branch :223-229).
 * out = (any(x < 0) | any(x > 1)) ? sigmoid(x) : x, decided per call over the whole buffer, no host sync.
 * `flag_scratch` is a 4-byte device word owned by the caller (zeroed internally with cudaMemsetAsync).
 * out may alias preds.  Math in fp32 (fp64 for MB200_F64), rounded to the storage dtype like ATen.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_curve_sigmoid_if_logits(const void* preds, int dtype, int64_t n, void* out,
                                            uint32_t* flag_scratch, void* stream);
/* softmax(dim=1) variant for [n, num_classes] row-major scores (multiclass curve metrics,
 * functional/classification/precision_recall_curve.py:454). */
/* mb200_curve_softmax_if_logits with a caller-owned scratch of 8 + n bytes (4-byte aligned, contents irrelevant; a shorter or
 * unaligned scratch takes the original kernels with its first aligned word as the vote word): rows of at
 * most 1024 f32 / f16 / bf16 scores are read ONCE (row kept in registers, one `expf` per score); a row that itself holds a score
 * outside [0, 1] writes its softmax, the others are written through and revisited by a second (normally empty) launch only when
 * the batch turned out to be logits.  Same bits as mb200_curve_softmax_if_logits. */
MB200_API int mb200_curve_softmax_if_logits_scratch(const void* preds, int dtype, int64_t n, int64_t num_classes, void* out,
                                                    void* scratch, int64_t scratch_bytes, void* stream);
/* mb200_curve_sigmoid_if_logits with a caller-owned scratch of mb200_curve_normalize_scratch_bytes(n) bytes (4-byte aligned,
 * contents irrelevant; an unaligned scratch takes the original kernels with its first aligned word as the vote word): large 16-byte aligned f32 / f16 / bf16 batches are then read ONCE — every 16 KB tile that itself
 * holds a score outside [0, 1] knows the vote and writes sigmoids, the others write the scores through and are revisited by a
 * second (normally empty) launch only when the batch turned out to be logits. */
MB200_API int64_t mb200_curve_normalize_scratch_bytes(int64_t n);
MB200_API int mb200_curve_sigmoid_if_logits_scratch(const void* preds, int dtype, int64_t n, void* out, void* scratch,
                                                    int64_t scratch_bytes, void* stream);
MB200_API int mb200_curve_softmax_if_logits(const void* preds, int dtype, int64_t n, int64_t num_classes, void* out,
                                            uint32_t* flag_scratch, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K3/K5 — exact-mode curve evaluation: sort + tie-collapsing TP/FP scan + AUROC / average precision.
 * Replaces functional/classification/precision_recall_curve.py:30-82 (_binary_clf_curve), roc.py:40-80,
 * auroc.py:83-107 (max_fpr=None), average_precision.py:70-75, utilities/compute.py:101-109, and for
 * num_classes > 1 the per-class Python loops of roc.py:176-181 / precision_recall_curve.py:565-569
 * (one segment per class, sorted together in one batched radix sort).
 *
 *  preds      : num_classes == 1: [n] scores; else [n, num_classes] row-major.  f32 / f16 / bf16.
 *  target     : [n] integer labels.  Positive for curve c: target == c (num_classes == 1: target == pos_label).
 *  workspace  : device scratch of at least mb200_curve_workspace_bytes(num_classes, n) bytes
 *  out_auroc  : float32 [num_classes]   area under ROC (0 when a curve has no positives or no negatives)
 *  out_ap     : float32 [num_classes]   average precision (-0.0 when a curve has no positives, like the reference)
 *  out_counts : int64 [num_classes][3]  {#positives, #negatives, #distinct thresholds U}
 *  fps_out, tps_out, thr_out : optional (all or none) float32 [num_classes][n]; for curve c the first U entries
 *               are the reference's `fps, tps, thresholds` (descending thresholds), the rest is untouched.
 *  err_flag   : optional device word; MB200_FLAG_SPIN_TIMEOUT is raised if the sort's bounded look-back wait expires
 * TP/FP are counted in integers (n < 2^30 samples per curve); AUROC = exact integer sum / (2 P N) evaluated in fp64;
 * AP accumulated in fp64 in a fixed order (bitwise reproducible run to run).
 * ------------------------------------------------------------------------------------------------ */
MB200_API int64_t mb200_curve_workspace_bytes(int64_t num_classes, int64_t n);
/* float64 scores are sorted as 64-bit keys (the reference sorts them as doubles: functional/classification/
 * precision_recall_curve.py:60 `argsort`), 8 radix passes and a larger workspace: size it with the score dtype.  For f64
 * scores `thr_out` of the evaluate calls is double [num_classes][n]; for every other score type float [num_classes][n]
 * (half / bfloat16 scores are compared as float32, like ATen). fps / tps stay float32 (the reference's `target * 1.0`). */
MB200_API int64_t mb200_curve_workspace_bytes_for(int64_t num_classes, int64_t n, int preds_dtype);
/* the packing step alone: class-major keys [num_classes][n] of [n, num_classes] scores, and sort+scan on packed keys
 * (positives of curve s: target == first_class + s; `keys` is sorted in place).  Used by the class-sharded multi-GPU
 * evaluation, which exchanges key rows between ranks (all-to-all) between the two calls. */
MB200_API int mb200_curve_pack_keys(const void* preds, int preds_dtype, int64_t n, int64_t num_classes,
                                    uint32_t* keys_out, void* stream);
MB200_API int mb200_curve_evaluate_keys(uint32_t* keys, const void* target, int target_dtype, int64_t n,
                                        int64_t segments, int64_t first_class, void* workspace, int64_t workspace_bytes,
                                        float* out_auroc, float* out_ap, int64_t* out_counts, uint32_t* err_flag,
                                        void* stream);
/* mb200_curve_evaluate_keys for keys of non-negative (or NaN) scores (metric states): the label is folded into bit 0 of the key
 * in place, 4-byte sort records; a key of a negative score raises MB200_FLAG_PREDS_RANGE (see mb200_curve_evaluate_nonneg). */
MB200_API int mb200_curve_evaluate_keys_nonneg(uint32_t* keys, const void* target, int target_dtype, int64_t n,
                                        int64_t segments, int64_t first_class, void* workspace, int64_t workspace_bytes,
                                        float* out_auroc, float* out_ap, int64_t* out_counts, uint32_t* err_flag,
                                        void* stream);
MB200_API int mb200_curve_evaluate(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                   int64_t n, int64_t num_classes, int64_t pos_label, void* workspace,
                                   int64_t workspace_bytes, float* out_auroc, float* out_ap, int64_t* out_counts,
                                   float* fps_out, float* tps_out, void* thr_out, uint32_t* err_flag, void* stream);
/* `_binary_clf_curve` with `sample_weights` (functional/classification/precision_recall_curve.py:64, 73-78): at every
 * distinct score (descending) tps = cumsum(w * [target == pos_label]), fps = cumsum(w * [target != pos_label]), accumulated
 * in fp64 in a fixed order.  weights: double [n].  fps_out / tps_out: double [n]; thr_out: double [n] for f64 scores, float
 * [n] otherwise; count_out: device int64, number of distinct thresholds (valid prefix of the three outputs). */
MB200_API int64_t mb200_curve_weighted_workspace_bytes(int64_t n, int preds_dtype);
MB200_API int mb200_curve_weighted_clf_curve(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                             const double* weights, int64_t n, int64_t pos_label, void* workspace,
                                             int64_t workspace_bytes, double* fps_out, double* tps_out, void* thr_out,
                                             int64_t* count_out, uint32_t* err_flag, void* stream);
/* mb200_curve_evaluate for scores PROMISED to be non-negative or NaN (in particular the output of normalize_logits_if_needed
 * — every state of the curve metric classes): 31-bit keys, the label rides in bit 0, the radix passes move 4-byte keys only.
 * A negative score (-0 is fine) raises MB200_FLAG_PREDS_RANGE in err_flag (results invalid).  float64 scores take the general
 * path. */
MB200_API int mb200_curve_evaluate_nonneg(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                        int64_t n, int64_t num_classes, int64_t pos_label, void* workspace,
                                        int64_t workspace_bytes, float* out_auroc, float* out_ap, int64_t* out_counts,
                                        float* fps_out, float* tps_out, void* thr_out, uint32_t* err_flag, void* stream);
/* Multilabel task: `num_labels` independent binary curves in one batched sort + scan.  preds / target are
 * [n, num_labels] row-major, positives are target == 1.  With has_ignore, entries with target == ignore_index are
 * removed from their own label's curve only (they are given the largest sort key and the scan stops before them).
 * Replaces the per-label Python loop of functional/classification/precision_recall_curve.py:822-834
 * (_multilabel_precision_recall_curve_compute), roc.py:_multilabel_roc_compute, auroc.py:308-333 and
 * average_precision.py:_multilabel_average_precision_compute.  Outputs as in mb200_curve_evaluate. */
MB200_API int mb200_curve_evaluate_multilabel(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                              int64_t n, int64_t num_labels, int has_ignore, int64_t ignore_index,
                                              void* workspace, int64_t workspace_bytes, float* out_auroc, float* out_ap,
                                              int64_t* out_counts, float* fps_out, float* tps_out, void* thr_out,
                                              uint32_t* err_flag, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K8 — COCO-style bounding-box mAP / mAR evaluation on the device.
 * Replaces detection/mean_ap.py:521-598 (MeanAveragePrecision.compute): the per-element host marshalling of
 * :867-958 and the third-party pycocotools calls at :538-546 (COCOeval.evaluate / accumulate and maskApi.c:bbIou;
 * algorithm restated with citations in oracle/coco_map.py).  `summarize` (means over the precision / recall tensors)
 * is left to the caller.
 *
 * Inputs are the concatenation of all images (list position = image id):
 *  det_box_xywh [n_det,4] f32, det_score [n_det] f32, det_label [n_det] i64, det_off [n_img+1] i32 (prefix counts)
 *  gt_box_xywh  [n_gt,4]  f32, gt_label [n_gt] i64, gt_crowd [n_gt] u8, gt_area [n_gt] f64 (<= 0: use w*h),
 *  gt_off [n_img+1] i32;  max_det_per_img / max_gt_per_img: largest per-image counts (sizes the shared-memory stage)
 *  classes [num_classes] i64 sorted unique labels over detections and ground truths; micro != 0: one class for all.
 *  iou_thr_host [n_iou_thr <= 16] f64 (HOST), rec_thr_dev [n_rec_thr] f64 (DEVICE), max_dets_host [n_max_dets <= 8]
 *  i64 ascending (HOST).
 * Outputs (device, f64), K = micro ? 1 : num_classes, A = 4 area ranges (all, small, medium, large):
 *  precision [T, R, K, A, M], recall [T, K, A, M], scores [T, R, K, A, M]; -1 where COCOeval leaves -1.
 * err_flag: optional device word; MB200_FLAG_CAPACITY is set when one image holds more than 256 ground truths of one
 * class.  Returns MB200_ERR_UNSUPPORTED when an image is too large for the shared-memory stage.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int64_t mb200_coco_map_workspace_bytes(int64_t n_det, int64_t num_classes, int64_t num_max_dets);
MB200_API int mb200_coco_map_evaluate(
    const float* det_box_xywh, const float* det_score, const int64_t* det_label, const int32_t* det_off,
    const float* gt_box_xywh, const int64_t* gt_label, const uint8_t* gt_crowd, const double* gt_area,
    const int32_t* gt_off, int64_t n_img, int64_t n_det, int64_t n_gt, int64_t max_det_per_img, int64_t max_gt_per_img,
    const int64_t* classes, int64_t num_classes, int micro, const double* iou_thr_host, int64_t n_iou_thr,
    const double* rec_thr_dev, int64_t n_rec_thr, const int64_t* max_dets_host, int64_t n_max_dets, void* workspace,
    int64_t workspace_bytes, double* precision, double* recall, double* scores, uint32_t* err_flag, void* stream);
/* The two phases of mb200_coco_map_evaluate on their own, for an evaluation sharded over ranks (detection/mean_ap.py
 * `_compute_distributed`; the reference gathers every image to every rank, mean_ap.py:1032-1063, and every rank evaluates
 * everything).  mb200_coco_map_match = COCOeval.evaluateImg for THIS rank's images: per detection (image order) the class
 * index in `classes` (int32), its rank inside its (image, class) (int32), and 64-bit match / ignore words (bit = area * T +
 * threshold); `npig` int32 [num_classes][4] is ADDED to (zero it first).  mb200_coco_map_accumulate = COCOeval.accumulate for
 * the classes [class_lo, class_hi) over records from ALL ranks (ties in score keep the order the records are given in):
 * precision / recall / scores are full-size [.., num_classes, ..] arrays, filled with -1 here, owned classes written. */
MB200_API int mb200_coco_map_match(const float* det_box_xywh, const float* det_score, const int64_t* det_label,
                                   const int32_t* det_off, const float* gt_box_xywh, const int64_t* gt_label,
                                   const uint8_t* gt_crowd, const double* gt_area, const int32_t* gt_off, int64_t n_img,
                                   int64_t max_det_per_img, int64_t max_gt_per_img, const int64_t* classes,
                                   int64_t num_classes, const double* iou_thr_host, int64_t n_iou_thr, int64_t max_det_last,
                                   int32_t* det_cat, int32_t* det_rank, uint64_t* det_match, uint64_t* det_ignore,
                                   int32_t* npig, uint32_t* err_flag, void* stream);
/* mb200_coco_map_match with what `iou_type="segm"` needs (reference detection/mean_ap.py:527-547 evaluation per IoU type,
 * :848-853 masks, :917-944 annotation areas):
 *   pair_inter     NULL = boxes.  Else instance masks: per image the [detections x ground truths] table of intersection pixel
 *                  counts (mb200_mask_pair_intersections), `pair_off` [n_img] its offsets, `det_mask_area` / `gt_mask_area`
 *                  the masks' pixel counts; IoU = inter / union as maskApi.c:rleIou (0 when inter is 0; crowd: union = the
 *                  detection's area), detections' area ranges from `det_mask_area`; the boxes are not read.
 *   gt_area_exact  `gt_area` is the annotation's final "area" (no w*h fallback for values <= 0).
 *   micro          every label is class 0 (npig then has one row). */
MB200_API int mb200_coco_map_match_ex(const float* det_box_xywh, const float* det_score, const int64_t* det_label,
                                      const int32_t* det_off, const float* gt_box_xywh, const int64_t* gt_label,
                                      const uint8_t* gt_crowd, const double* gt_area, const int32_t* gt_off, int64_t n_img,
                                      int64_t max_det_per_img, int64_t max_gt_per_img, const int64_t* classes,
                                      int64_t num_classes, int micro, const double* iou_thr_host, int64_t n_iou_thr,
                                      int64_t max_det_last, const double* pair_inter, const int64_t* pair_off,
                                      const double* det_mask_area, const double* gt_mask_area, int gt_area_exact,
                                      int32_t* det_cat, int32_t* det_rank, uint64_t* det_match, uint64_t* det_ignore,
                                      int32_t* npig, uint32_t* err_flag, void* stream);
MB200_API int mb200_coco_map_accumulate(const int32_t* det_cat, const float* det_score, const int32_t* det_rank,
                                        const uint64_t* det_match, const uint64_t* det_ignore, int64_t n_det,
                                        const int32_t* npig, int64_t num_classes, int64_t class_lo, int64_t class_hi,
                                        int64_t n_iou_thr, const double* rec_thr_dev, int64_t n_rec_thr,
                                        const int64_t* max_dets_host, int64_t n_max_dets, void* workspace,
                                        int64_t workspace_bytes, double* precision, double* recall, double* scores,
                                        uint32_t* err_flag, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K2 — binary / multilabel stat scores and confusion-matrix counts.
 * Replaces functional/classification/stat_scores.py:95-134 (_binary_stat_scores_format/_update), :681-714
 * (multilabel), confusion_matrix.py:119-152 and :477-516 (the 2x2 matrices are [[tn, fp], [fn, tp]]).
 *
 *  preds   : [n_outer, num_labels, inner] contiguous; floating scores (sigmoid applied when ANY value of the call
 *            lies outside [0,1], then `> threshold` with the threshold rounded to the score dtype, double -> float ->
 *            half / bfloat16, as ATen rounds a Python scalar) or integer labels compared raw against the target.
 *  target  : same layout, integer; elements equal to ignore_index are skipped; values outside {0,1} are skipped and
 *            flagged (MB200_FLAG_TARGET_RANGE); integer preds outside {0,1} are flagged (MB200_FLAG_PREDS_RANGE).
 *  counts  : int64 [G][4] += (tp, fp, tn, fn), G = num_labels, or n_outer * num_labels when samplewise != 0.
 *  flag_scratch : 4-byte device word (required for floating preds).
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_binary_stat_counts(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                       int64_t n_outer, int64_t num_labels, int64_t inner, double threshold,
                                       int has_ignore_index, int64_t ignore_index, int samplewise, int64_t* counts,
                                       uint32_t* flag_scratch, uint32_t* err_flag, void* stream);
/* Same contract with a larger caller-owned scratch (>= MB200_BINARY_SCRATCH_BYTES, 8-byte aligned, contents irrelevant): the
 * binary task (num_labels == 1, global counts, int64 targets, 16-byte aligned f32/f16/bf16 scores) then reads the scores ONCE,
 * counting under both outcomes of the batch-global logits vote and adding the selected set in a one-warp epilogue — 12 instead
 * of 16 bytes of traffic per element; every other shape takes the kernels of mb200_binary_stat_counts (a single-pass variant of
 * the multilabel column kernel was measured slower than its two passes at [2^20, 64] and removed). */
#define MB200_BINARY_SCRATCH_BYTES 128
MB200_API int mb200_binary_stat_counts_scratch(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                               int64_t n_outer, int64_t num_labels, int64_t inner, double threshold,
                                               int has_ignore_index, int64_t ignore_index, int samplewise, int64_t* counts,
                                               uint32_t* scratch, int64_t scratch_bytes, uint32_t* err_flag, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K9 — regression running sums (one fused map-reduce per update).
 * Replaces the `_x_update` functions of functional/regression/{mse,mae,mape,symmetric_mape,wmape,log_mse,log_cosh,
 * minkowski,r2,explained_variance,tweedie_deviance}.py (file:line list in csrc/regression.cu).
 *  preds, target : [n, d] contiguous, same floating dtype (d = num_outputs; flatten to d = 1 for scalar metrics)
 *  op            : 0 MSE sum d^2 | 1 MAE sum|d| | 2 MAPE sum|d|/max(|t|,eps) | 3 SMAPE sum|d|/max(|t|+|p|,eps)
 *                  4 WMAPE {sum|d|, sum|t|} | 5 MSLE sum(log1p p - log1p t)^2 | 6 LogCosh sum log((e^d+e^-d)/2)
 *                  7 Minkowski sum|d|^param | 8 R2/RSE {sum t^2, sum t, sum (t-p)^2}
 *                  9 ExplainedVariance {sum (t-p), sum (t-p)^2, sum t, sum t^2}          (d = p - t)
 *                  10 Tweedie deviance of power `param` (1 Poisson, 2 Gamma, else the general form; 0 is op 0) with the
 *                     domain census the reference gets from extra passes: {sum dev, #(p <= 0), #(t < 0), #(t == 0)}
 *  out_sums      : float64 [num_sums(op)][d], overwritten
 *  scratch       : float64 [mb200_regression_scratch_doubles(n, d, op)]
 * Terms are evaluated in fp32 (fp64 for fp64 inputs), sums in fp64 with a fixed order (bitwise reproducible).
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_regression_num_sums(int op);
MB200_API int64_t mb200_regression_scratch_doubles(int64_t n, int64_t d, int op);
MB200_API int mb200_regression_sums(const void* preds, const void* target, int dtype, int64_t n, int64_t d, int op,
                                    double param, double epsilon, double* out_sums, double* scratch, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K4 — binned (fixed-threshold) curve state update.
 * Replaces functional/classification/precision_recall_curve.py:191-251 (binary) and :464-533 (multiclass):
 * the multi-threshold confusion matrix confmat[i, (c,) target, score >= thr[i]].
 *  preds      : [n] (num_classes == 1) or [n, num_classes] row-major scores, already sigmoid/softmax-normalised
 *  target     : [n] integer labels; binary: 1 = positive, 0 = negative, anything else skipped
 *  thresholds_sorted : [num_thresholds] of dtype `thresholds_dtype` (any float or integer tag but bool), ASCENDING (device)
 *  compare_dtype : the float dtype tag D in which `score >= threshold` is evaluated: the score dtype, F32 or F64 (the
 *                  score dtype when that is F64).  mb200_binned_curve_compare_dtype gives the reference's choice.
 *  confmat    : int64 [num_thresholds, num_classes, 2, 2] (binary callers view it as [T, 2, 2]), updated in place
 *  scratch    : uint64 [mb200_binned_curve_scratch_words(...)], zero on entry, left zeroed (self-cleaning)
 * ------------------------------------------------------------------------------------------------ */
MB200_API int64_t mb200_binned_curve_scratch_words(int64_t num_classes, int64_t num_thresholds);
/* The dtype tag in which the reference compares one update of n rows (after the ignore_index filter): the score dtype on its
 * loop branch (binary: n > 50 000; multiclass: n * num_classes^2 > 10^6), else the promotion of score and threshold dtypes
 * (multilabel always).  -1 for a score or threshold tag that is not accepted. */
MB200_API int mb200_binned_curve_compare_dtype(int preds_dtype, int thresholds_dtype, int64_t n, int64_t num_classes,
                                               int multilabel);
MB200_API int mb200_binned_curve_update(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                        int64_t n, int64_t num_classes, const void* thresholds_sorted, int thresholds_dtype,
                                        int compare_dtype, int64_t num_thresholds, int64_t* confmat, uint64_t* scratch,
                                        void* stream);
/* Multilabel variant (replaces precision_recall_curve.py:745-799 _multilabel_precision_recall_curve_format + _update):
 * target is [n, num_labels] like preds; entries whose target is neither 0 nor 1, or (has_ignore_index != 0) equals
 * ignore_index reduced to the target dtype's width, are skipped.  confmat: int64 [num_thresholds, num_labels, 2, 2]. */
MB200_API int mb200_binned_curve_update_multilabel(const void* preds, int preds_dtype, const void* target,
                                                   int target_dtype, int64_t n, int64_t num_labels,
                                                   const void* thresholds_sorted, int thresholds_dtype, int compare_dtype,
                                                   int64_t num_thresholds, int has_ignore_index, int64_t ignore_index,
                                                   int64_t* confmat, uint64_t* scratch, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K11 — collection-level fusion (csrc/fused.cu): one pass over a shared [n, num_classes] batch for a multiclass stat-scores
 * metric AND an exact-mode multiclass curve metric of the same MetricCollection (collections.py:231-262 hands the batch to
 * every member; stat_scores.py:328-448 then runs argmax -> bincount and utilities/compute.py:190-229 the range vote + softmax).
 * tp/fp/tn/fn/workspace: as mb200_multiclass_stat_scores_update (top-1, global, no ignore_index).  probs_out [n, num_classes]
 * (same dtype as preds) receives what `normalize_logits_if_needed(preds, "softmax")` returns: the softmax when any score of
 * the batch lies outside [0, 1], else the scores themselves; logits_flag (device word, overwritten) holds that vote.
 * num_classes <= 1024 (a warp keeps a row in registers).
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_multiclass_stats_softmax_update(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                                    int64_t n, int64_t num_classes, int micro, int64_t* tp, int64_t* fp,
                                                    int64_t* tn, int64_t* fn, int64_t* workspace, void* probs_out,
                                                    uint32_t* logits_flag, uint32_t* err_flag, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K10 — cross-rank state exchange over NVLink peer memory (csrc/peer.cu).  One process per GPU; `peer_bases` is a DEVICE
 * array of `world` base pointers of one symmetric allocation (entry r = rank r's base, peer-mapped into this process).
 * Replaces the per-state `barrier + all_gather(shape) + all_gather(data)` of Metric._sync_dist / gather_all_tensors
 * (metric.py:501-540, utilities/distributed.py:100-153) for the states that shard naturally.  The entry points enqueue
 * stores / loads only: cross-rank ordering is the caller's (a signal-pad barrier on the same stream before the data is
 * consumed and before a region is reused).
 *
 * mb200_peer_pack_keys_put: the class-sharded exchange of one-vs-rest curve scores fused with key packing.  preds is this
 *   rank's [n_local, num_classes] score matrix; class c is owned by rank c / classes_per_rank, whose key matrix
 *   uint32 [classes_per_rank][n_total] starts `keys_offset_bytes` into its allocation; this rank's samples occupy columns
 *   [col_offset, col_offset + n_local).  Keys are the ones mb200_curve_pack_keys produces (ready for
 *   mb200_curve_evaluate_keys).
 * mb200_peer_put_all: copies `nbytes` from `src` to offset `dst_offset_bytes` of EVERY rank's allocation (all-gather by
 *   peer stores when every rank uses its own offset).
 * mb200_peer_reduce_put_i64: all-reduce of an int64 [n] state held at `in_offset_bytes` of every rank's allocation: this
 *   rank reduces its slice of every rank's input (op: 0 sum, 1 max, 2 min; bit-exact) and stores the result at
 *   `out_offset_bytes` of every rank's allocation.  Offsets must be 16-byte aligned; world <= 16.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_peer_pack_keys_put(const void* preds, int preds_dtype, int64_t n_local, int64_t num_classes,
                                       int64_t classes_per_rank, int world, int64_t n_total, int64_t col_offset,
                                       void* const* peer_bases, int64_t keys_offset_bytes, void* stream);
MB200_API int mb200_peer_put_all(const void* src, int64_t nbytes, void* const* peer_bases, int64_t dst_offset_bytes,
                                 int world, void* stream);
MB200_API int mb200_peer_reduce_put_i64(void* const* peer_bases, int64_t in_offset_bytes, int64_t out_offset_bytes,
                                        int64_t n, int rank, int world, int op, void* stream);

/* ---- K12: instance masks for MeanAveragePrecision(iou_type="segm") (csrc/maskiou.cu) --------------------------------------
 * The reference run-length encodes every mask on the host (detection/mean_ap.py:848-853, pycocotools mask_utils.encode) and
 * pycocotools intersects run-length codes pair by pair on the host (maskApi.c:rleIou).  Here:
 * mb200_mask_pack_bits: `masks` uint8/bool [n_masks][pixels_per_mask] (non-zero = set) -> one bit per pixel, 32 pixels per
 *   word in pixel order, row m at words_out + m * out_stride_words; area_out[m] = number of set pixels (int64).
 * mb200_mask_pair_intersections: for image i with detections [det_off[i], det_off[i+1]) and ground truths [gt_off[i],
 *   gt_off[i+1]), whose bit rows start at det_words + det_word_off[d] / gt_words + gt_word_off[g] and are img_words[i] words
 *   long: inter_out[pair_off[i] + d_local * G_i + g_local] = popcount(det & gt) as a double; pairs of different labels
 *   (unless micro) are written as 0 — the matcher never reads them.  max_pairs_per_img only sizes the grid. */
MB200_API int mb200_mask_pack_bits(const uint8_t* masks, int64_t n_masks, int64_t pixels_per_mask, uint32_t* words_out,
                                   int64_t out_stride_words, int64_t* area_out, void* stream);
/* The same packing straight into the per-image state entry of MeanAveragePrecision (one call per image and side at update()):
 * entry_out int32 [3 + n + n * ceil(H*W/32)] = [n, H, W, area_0 .. area_{n-1}, bit rows of the n masks]. */
MB200_API int mb200_mask_pack_entry(const uint8_t* masks, int64_t n_masks, int64_t height, int64_t width, int32_t* entry_out,
                                    void* stream);
MB200_API int mb200_mask_pair_intersections(const uint32_t* det_words, const int64_t* det_word_off, const uint32_t* gt_words,
                                            const int64_t* gt_word_off, const int32_t* det_off, const int32_t* gt_off,
                                            const int32_t* img_words, const int64_t* det_label, const int64_t* gt_label,
                                            int micro, const int64_t* pair_off, int64_t n_img, int64_t max_pairs_per_img,
                                            double* inter_out, void* stream);

/* ---- K13: per-row KL divergence (csrc/kldiv.cu) ------------------------------------------------------------------------------
 * Replaces `_kld_update` (functional/regression/kl_divergence.py:25-46): measures_out[i] = KL(p_i || q_i) for the rows of the
 * [n, d] distributions `p`, `q` (dtype tag f32/f16/bf16/f64, row-major, same dtype), in the inputs' dtype.  log_prob = 0: both
 * rows are normalised to sum 1 first and terms with p = 0 count 0 (`_safe_xlogy`, utilities/compute.py:32-44); log_prob = 1:
 * sum exp(p) * (p - q).  One read of p and q from HBM (the reference chain makes eight passes with [n, d] temporaries). */
MB200_API int mb200_kl_divergence_rows(const void* p, const void* q, int dtype, int64_t n, int64_t d, int log_prob,
                                       void* measures_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* METRICS_B200_H_ */
