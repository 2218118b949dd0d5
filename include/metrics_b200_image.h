/*
 * metrics_b200 — C-ABI of the windowed-moment image kernels (K20 SSIM, K21 VIF and UQI), exported from the same libmetrics_b200.so as
 * include/metrics_b200.h and following its conventions: device pointers, a CUDA stream handle as the last argument,
 * 0 or a negative MB200_ERR_* code returned, message in mb200_last_error().
 *
 * Reference replaced (paths relative to src/torchmetrics/):
 *   functional/image/ssim.py:113-186   data range, tuple clamp, reflect padding, the five-image cat, the grouped conv and
 *                                      the element-wise epilogue of _ssim_update, and the per-image means
 *   functional/image/ssim.py:402-413   the 2x2 (2-D) / 2x2x2 (3-D) average pool between the scales of MS-SSIM
 *   functional/image/vif.py:45-82      the VIF scale loop: decimation, the five dense convolutions, masks and sums
 *   functional/image/uqi.py:87-114     pad, five-image cat, grouped conv, epilogue and crop of UQI
 *
 * Geometry: every entry point takes 5-D inputs [b, c, d, h, w] with element strides (s_n, s_c, s_d, s_h, s_w).  A 2-D
 * batch [B, C, H, W] is d = 1, s_d = 0 with one depth tap and no depth pad; a 3-D batch [B, C, X, Y, Z] is d = X, h = Y,
 * w = Z.  preds_dtype is a float tag (MB200_F32 / F16 / BF16 / F64); target may be any float tag and is rounded to the
 * preds dtype on load.  Nothing here synchronises the host.
 */
#ifndef METRICS_B200_IMAGE_H_
#define METRICS_B200_IMAGE_H_

#include "metrics_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* consts[]: device float64 words written by mb200_ssim_data_range and read by mb200_ssim_update */
#define MB200_SSIM_RANGE 0 /* max(preds.max() - preds.min(), target.max() - target.min()) */
#define MB200_SSIM_C1 1    /* (k1 * range) ** 2 */
#define MB200_SSIM_C2 2    /* (k2 * range) ** 2 */
#define MB200_SSIM_CONSTS 3

/* per-axis tap count bounds; the filter's tile must also fit in shared memory (mb200_ssim_scratch_bytes returns -1) */
#define MB200_SSIM_MAX_TAPS 255

/* ------------------------------------------------------------------------------------------------
 * Bytes of scratch mb200_ssim_update and mb200_ssim_data_range need for this geometry (16-byte aligned, contents
 * irrelevant), or -1 when an argument is out of range or the filter does not fit in shared memory.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int64_t mb200_ssim_scratch_bytes(int preds_dtype, int64_t b, int64_t c, int64_t d, int64_t h, int64_t w,
                                           int taps_d, int taps_h, int taps_w, int pad_d, int pad_h, int pad_w);

/* ------------------------------------------------------------------------------------------------
 * Data-range pre-pass (data_range=None).  consts[MB200_SSIM_RANGE] = max(pmax - pmin, tmax - tmin) with Python's max
 * (the target range only when it is larger; NaN inside a tensor propagates as torch.max / torch.min do); the differences
 * are rounded to the preds dtype, c1 and c2 are computed in float32 (float64 for float64 preds).  b * c * d * h * w >= 1.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_ssim_data_range(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t b,
                                    int64_t c, int64_t d, int64_t h, int64_t w, int64_t preds_s_n, int64_t preds_s_c,
                                    int64_t preds_s_d, int64_t preds_s_h, int64_t preds_s_w, int64_t target_s_n,
                                    int64_t target_s_c, int64_t target_s_d, int64_t target_s_h, int64_t target_s_w,
                                    double k1, double k2, double* consts, void* scratch, int64_t scratch_bytes,
                                    void* stream);

/* ------------------------------------------------------------------------------------------------
 * K20 — SSIM of every image.  Output size per axis: o = n + 2 * pad - taps + 1 (>= 1).  Padding is reflect
 * (pad < n per axis).  weights: device [taps_d + taps_h + taps_w] in the preds dtype, the separable filter per axis.
 * clamp != 0 clamps both inputs to [clamp_lo, clamp_hi] on load.  consts: device [MB200_SSIM_CONSTS] from
 * mb200_ssim_data_range, or NULL to use c1 / c2.  Moments are taken about a per-tile shift, in float32 (float64 preds:
 * float64).
 *   sim[b]:  float64 mean of the SSIM map over channels and positions.
 *   cs[b]:   float64 mean of upper / lower over the crop [pad:o-pad] per axis (the depth axis too when crop_depth != 0);
 *            an axis with pad 0 makes the crop empty and cs NaN.  NULL: not computed.
 *   map:     NULL, or [b, c, o_d, o_h, o_w] contiguous in the preds dtype.
 * Per-image sums are float64 in a fixed order: results are identical from run to run.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_ssim_update(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t b,
                                int64_t c, int64_t d, int64_t h, int64_t w, int64_t preds_s_n, int64_t preds_s_c,
                                int64_t preds_s_d, int64_t preds_s_h, int64_t preds_s_w, int64_t target_s_n,
                                int64_t target_s_c, int64_t target_s_d, int64_t target_s_h, int64_t target_s_w, int taps_d,
                                int taps_h, int taps_w, int pad_d, int pad_h, int pad_w, int crop_depth,
                                const void* weights, int clamp, double clamp_lo, double clamp_hi, const double* consts,
                                double c1, double c2, double* sim, double* cs, void* map, void* scratch,
                                int64_t scratch_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * The next MS-SSIM scale: 2x2 (pool_depth == 0) or 2x2x2 average pool of both inputs, floor sizes, written contiguous
 * [b, c, d', h / 2, w / 2] in the preds dtype (d' = d / 2 when pool_depth, else d).  target is rounded to the preds
 * dtype first.  Every output size must be >= 1.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_ssim_avg_pool(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t b,
                                  int64_t c, int64_t d, int64_t h, int64_t w, int64_t preds_s_n, int64_t preds_s_c,
                                  int64_t preds_s_d, int64_t preds_s_h, int64_t preds_s_w, int64_t target_s_n,
                                  int64_t target_s_c, int64_t target_s_d, int64_t target_s_h, int64_t target_s_w,
                                  int pool_depth, void* preds_out, void* target_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K21 — one scale of pixel-domain VIF (functional/image/vif.py:53-82) on K20's moments, valid filtering (no pads, no
 * crop).  Output size per axis o = n - taps + 1 (>= 1).  weights: device [taps_d + taps_h + taps_w] in the preds dtype.
 * eps and sigma_n_sq: the reference's constants already rounded to the preds dtype.  Writes, per (image, channel) in
 * [b, c] order, the float64 sums over the scale's positions of
 *   preds_sum:   log10(1 + g² σt / (σv + σn²))    target_sum:   log10(1 + σt / σn²)
 * after the reference's masks (σt < eps, σp < eps, g < 0, σv clamped to eps, in that order).  Scratch:
 * mb200_ssim_scratch_bytes with zero pads.  Fixed summation order: results are identical from run to run.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_vif_scale_update(const void* preds, int preds_dtype, const void* target, int target_dtype,
                                     int64_t b, int64_t c, int64_t d, int64_t h, int64_t w, int64_t preds_s_n,
                                     int64_t preds_s_c, int64_t preds_s_d, int64_t preds_s_h, int64_t preds_s_w,
                                     int64_t target_s_n, int64_t target_s_c, int64_t target_s_d, int64_t target_s_h,
                                     int64_t target_s_w, int taps_d, int taps_h, int taps_w, const void* weights,
                                     double eps, double sigma_n_sq, double* preds_sum, double* target_sum,
                                     void* scratch, int64_t scratch_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * The next VIF scale: conv2d(x, k)[..., ::2, ::2] of both inputs, per depth plane, with the separable filter
 * weights [taps_h + taps_w] (preds dtype), written contiguous [b, c, d, ceil((h - taps_h + 1) / 2),
 * ceil((w - taps_w + 1) / 2)] in the preds dtype.  taps <= size per axis.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_vif_decimate(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t b,
                                 int64_t c, int64_t d, int64_t h, int64_t w, int64_t preds_s_n, int64_t preds_s_c,
                                 int64_t preds_s_d, int64_t preds_s_h, int64_t preds_s_w, int64_t target_s_n,
                                 int64_t target_s_c, int64_t target_s_d, int64_t target_s_h, int64_t target_s_w,
                                 int taps_h, int taps_w, const void* weights, void* preds_out, void* target_out,
                                 void* stream);

/* ------------------------------------------------------------------------------------------------
 * K21 — universal image quality index (functional/image/uqi.py:94-114) on K20's moments: reflect pads and taps as for
 * mb200_ssim_update, the map ((2 μx μy) 2σxy) / ((μx² + μy²)(σx² + σy²) + eps) with eps the preds dtype's machine
 * epsilon.  sums[b]: float64 sum of the map over [crop_h : o_h - crop_h] x [crop_w : o_w - crop_w] of every channel and
 * depth (a zero margin gives an empty crop and a zero sum).  map: NULL, or [b, c, o_d, o_h, o_w] contiguous in the
 * preds dtype.  Scratch: mb200_ssim_scratch_bytes.
 * ------------------------------------------------------------------------------------------------ */
MB200_API int mb200_uqi_update(const void* preds, int preds_dtype, const void* target, int target_dtype, int64_t b,
                               int64_t c, int64_t d, int64_t h, int64_t w, int64_t preds_s_n, int64_t preds_s_c,
                               int64_t preds_s_d, int64_t preds_s_h, int64_t preds_s_w, int64_t target_s_n,
                               int64_t target_s_c, int64_t target_s_d, int64_t target_s_h, int64_t target_s_w, int taps_d,
                               int taps_h, int taps_w, int pad_d, int pad_h, int pad_w, int crop_h, int crop_w,
                               const void* weights, double eps, double* sums, void* map, void* scratch,
                               int64_t scratch_bytes, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* METRICS_B200_IMAGE_H_ */
