"""CPU and GPU: every C entry point that takes a score dtype tag, called directly through `_native.lib()`; for K16's group
sort that is its graded target, for K18 and K19 their label maps.  Where an entry point takes two tags, one is held fixed.

A tag the entry point does not accept must come back with its own error code and message before any CUDA work: no launch is
counted and, on a box without a GPU, no CUDA error masks the dtype error.  On such a box every accepted tag must get past the
tag-to-type dispatch to the first CUDA call (code -2), so a type dropped from a dispatch fails here.  With a CUDA device the
buffers are device memory and only rejected tags are driven, so nothing is launched."""
import pytest
import torch

from metrics_b200 import _native

F32, F16, BF16, F64, I64 = _native.F32, _native.F16, _native.BF16, _native.F64, _native.I64
FLOAT = {F32, F16, BF16, F64}
FLOAT_NO_F64 = {F32, F16, BF16}
LABELS = {_native.I64, _native.I32, _native.I16, _native.I8, _native.U8, _native.BOOL}
TAGS = [-1] + list(range(10)) + [10]  # every mb200_dtype and one past either end

INVALID, UNSUPPORTED = -1, -3
N, C = 16, 3
BIG_N = 40000  # above the one-CTA sigmoid path: takes the large-batch and speculative paths
NBYTES = 1 << 20


class _Buffers(dict):
    """`b.name` is the address of a zeroed NBYTES buffer, allocated on first use and kept for the module's lifetime: device
    memory when a GPU is present, host memory otherwise."""

    def __getattr__(self, name):
        if name not in self:
            self[name] = torch.zeros(NBYTES, dtype=torch.uint8, device="cuda" if torch.cuda.is_available() else "cpu")
        return self[name].data_ptr()


_BUF = _Buffers()

FLOAT_MSG = "scores must be floating point (dtype tag %d)"
SOFTMAX_MSG = "softmax scores must be f32/f16/bf16/f64 (dtype tag %d)"
SCORES4_MSG = "scores must be f32/f16/bf16/f64 (dtype tag %d)"
SCORES3_MSG = "scores must be f32/f16/bf16 (dtype tag %d)"
CLASS_DIM_MSG = "preds with a class dimension must be floating point (got dtype tag %d)"
REGRESSION_MSG = "regression inputs must be floating point (dtype tag %d)"


def _curve(fn, b, d):
    return fn(b.p, d, b.t, I64, N, 1, 1, b.ws, NBYTES, b.auroc, b.ap, b.counts, None, None, None, b.err, 0)


def _hausdorff(L, b, d, input_format):
    """Two 4 x 4 images of C classes, int64 target, read through their strides (the class stride is ignored for index labels),
    every pair in one launch."""
    s = (C * 16, 16, 4, 1)
    return L.mb200_hausdorff_distance(b.p, d, b.t, I64, input_format, 2, C, 4, 4, *s, *s, 0, 0, 0, 1.0, 1.0, 0, 2 * C, b.out, b.ws,
                                      NBYTES, b.err, 0)


# name -> (accepted tags, error code, error message format, call(lib, buffers, tag) -> return code)
ENTRIES = {
    "sigmoid_small": (FLOAT, INVALID, FLOAT_MSG, lambda L, b, d: L.mb200_curve_sigmoid_if_logits(b.p, d, N, b.out, b.flag, 0)),
    "sigmoid_large": (FLOAT, INVALID, FLOAT_MSG,
                      lambda L, b, d: L.mb200_curve_sigmoid_if_logits(b.p, d, BIG_N, b.out, b.flag, 0)),
    "sigmoid_scratch": (FLOAT, INVALID, FLOAT_MSG,
                        lambda L, b, d: L.mb200_curve_sigmoid_if_logits_scratch(b.p, d, BIG_N, b.out, b.ws, NBYTES, 0)),
    "softmax": (FLOAT, INVALID, SOFTMAX_MSG, lambda L, b, d: L.mb200_curve_softmax_if_logits(b.p, d, N, C, b.out, b.flag, 0)),
    "softmax_scratch": (FLOAT, INVALID, SOFTMAX_MSG,
                        lambda L, b, d: L.mb200_curve_softmax_if_logits_scratch(b.p, d, N, C, b.out, b.ws, NBYTES, 0)),
    "curve_evaluate": (FLOAT, UNSUPPORTED, SCORES4_MSG, lambda L, b, d: _curve(L.mb200_curve_evaluate, b, d)),
    "curve_evaluate_nonneg": (FLOAT, UNSUPPORTED, SCORES4_MSG, lambda L, b, d: _curve(L.mb200_curve_evaluate_nonneg, b, d)),
    "curve_evaluate_multilabel": (FLOAT, UNSUPPORTED, SCORES4_MSG, lambda L, b, d: L.mb200_curve_evaluate_multilabel(
        b.p, d, b.t, I64, N, C, 1, -1, b.ws, NBYTES, b.auroc, b.ap, b.counts, None, None, None, b.err, 0)),
    "curve_pack_keys": (FLOAT_NO_F64, UNSUPPORTED, SCORES3_MSG, lambda L, b, d: L.mb200_curve_pack_keys(b.p, d, N, C, b.out, 0)),
    "curve_weighted": (FLOAT, UNSUPPORTED, SCORES4_MSG, lambda L, b, d: L.mb200_curve_weighted_clf_curve(
        b.p, d, b.t, I64, b.weights, N, 1, b.ws, NBYTES, b.fps, b.tps, b.thr, b.counts, b.err, 0)),
    # binary counts read every tag that is not floating as integer predictions: none is rejected
    "binary_counts": (FLOAT | LABELS, None, None, lambda L, b, d: L.mb200_binary_stat_counts(
        b.p, d, b.t, I64, N, 1, 1, 0.5, 0, 0, 0, b.out, b.flag, b.err, 0)),
    "binary_counts_scratch": (FLOAT | LABELS, None, None, lambda L, b, d: L.mb200_binary_stat_counts_scratch(
        b.p, d, b.t, I64, N, 1, 1, 0.5, 0, 0, 0, b.out, b.flag, 72, b.err, 0)),
    "regression": (FLOAT, INVALID, REGRESSION_MSG,
                   lambda L, b, d: L.mb200_regression_sums(b.p, b.t, d, N, 1, 0, 0.0, 0.0, b.out, b.ws, 0)),
    "regression_columns": (FLOAT, INVALID, REGRESSION_MSG,
                           lambda L, b, d: L.mb200_regression_sums(b.p, b.t, d, N, C, 0, 0.0, 0.0, b.out, b.ws, 0)),
    "confmat": (FLOAT, INVALID, CLASS_DIM_MSG, lambda L, b, d: L.mb200_multiclass_confmat_update(
        b.p, d, 1, b.t, I64, N, C, 1, 0, 0, b.out, b.err, 0)),
    "confmat_labels": (LABELS, INVALID, "label-format preds must have an integer dtype (got dtype tag %d)",
                       lambda L, b, d: L.mb200_multiclass_confmat_update(b.p, d, 0, b.t, I64, N, C, 1, 0, 0, b.out, b.err, 0)),
    "stat_scores": (FLOAT, INVALID, CLASS_DIM_MSG, lambda L, b, d: L.mb200_multiclass_stat_scores_update(
        b.p, d, 1, b.t, I64, N, C, 1, 0, 0, 0, b.tp, b.fp, b.tn, b.fn, b.ws, b.err, 0)),
    "stat_scores_samplewise": (FLOAT, INVALID, CLASS_DIM_MSG, lambda L, b, d: L.mb200_multiclass_stat_scores_samplewise(
        b.p, d, 1, b.t, I64, N, C, 1, 0, 0, b.out, b.counts, b.err, 0)),
    "stat_scores_topk": (FLOAT, INVALID, "top-k needs floating scores (dtype tag %d)",
                         lambda L, b, d: L.mb200_multiclass_stat_scores_topk_update(
                             b.p, d, b.t, I64, N, C, 2, 0, 0, b.tp, b.fp, b.tn, b.fn, b.ws, b.err, 0)),
    "argmax": (FLOAT, INVALID, CLASS_DIM_MSG, lambda L, b, d: L.mb200_argmax_rows(b.p, d, N, C, 1, b.out, 0)),
    "stats_softmax": (FLOAT_NO_F64, INVALID, SCORES3_MSG, lambda L, b, d: L.mb200_multiclass_stats_softmax_update(
        b.p, d, b.t, I64, N, C, 0, b.tp, b.fp, b.tn, b.fn, b.ws, b.out, b.flag, b.err, 0)),
    # K4 with float32 thresholds compared in float64, and (multilabel) uint8-wrapped ignore_index 257
    "binned_dtypes": (FLOAT, INVALID, FLOAT_MSG,
                      lambda L, b, d: L.mb200_binned_curve_update(b.p, d, b.t, I64, N, 1, b.thr, F32, F64, 5, b.out, b.ws, 0)),
    "binned_multilabel_dtypes": (FLOAT, INVALID, FLOAT_MSG, lambda L, b, d: L.mb200_binned_curve_update_multilabel(
        b.p, d, b.t, I64, N, C, b.thr, F32, F64, 5, 1, 257, b.out, b.ws, 0)),
    # the thresholds' tag is the one varied: any float or integer list
    "binned_thresholds": (FLOAT | LABELS - {_native.BOOL}, INVALID, "thresholds must be floating point or integer (dtype tag %d)",
                          lambda L, b, d: L.mb200_binned_curve_update(b.p, F32, b.t, I64, N, 1, b.thr, d, F64, 5, b.out, b.ws, 0)),
    "binned_multilabel_thresholds": (FLOAT | LABELS - {_native.BOOL}, INVALID,
                                     "thresholds must be floating point or integer (dtype tag %d)",
                                     lambda L, b, d: L.mb200_binned_curve_update_multilabel(
                                         b.p, F32, b.t, I64, N, C, b.thr, d, F64, 5, 0, 0, b.out, b.ws, 0)),
    "kl_divergence": (FLOAT, INVALID, "distributions must be f32/f16/bf16/f64 (dtype tag %d)",
                      lambda L, b, d: L.mb200_kl_divergence_rows(b.p, b.t, d, N, C, 0, b.out, 0)),
    "peer_pack_keys_put": (FLOAT_NO_F64, INVALID, SCORES3_MSG,
                           lambda L, b, d: L.mb200_peer_pack_keys_put(b.p, d, N, C, 2, 2, 2 * N, 0, b.peers, 0, 0)),
    "calibration_top_label": (FLOAT, INVALID, "preds must be f32/f16/bf16/f64 (dtype tag %d)",
                              lambda L, b, d: L.mb200_calibration_top_label(
                                  b.p, d, b.t, I64, N, C, 0, 0, b.out, b.acc, b.ws, NBYTES, b.err, 0)),
    "calibration_bin_sums": (FLOAT, INVALID, "confidences must be f32/f16/bf16/f64 (dtype tag %d)",
                             lambda L, b, d: L.mb200_calibration_bin_sums(
                                 b.p, d, b.t, I64, N, b.thr, 10, b.counts, b.fps, b.tps, b.ws, NBYTES, 0)),
    # one-hot [2, C, N] planar inputs sharing the tag, op 1 (the product)
    "segmentation_one_hot": (FLOAT_NO_F64 | LABELS, INVALID, "unsupported dtype tag %d",
                             lambda L, b, d: L.mb200_segmentation_overlap_counts(
                                 b.p, d, b.t, d, 2, C, N, 1, 0, C * N, C * N, 1, 0, b.out, b.ws, NBYTES, b.err, 0)),
    # the target's tag is the one varied
    "retrieval_sort": ({I64, F32}, INVALID, "target must be int64 or float32 (dtype tag %d)", lambda L, b, d: L.mb200_retrieval_sort(
        b.idx, b.p, b.t, d, N, 0, 0, b.sort_keys, b.out, b.offsets, b.info, b.ws, NBYTES, 0)),
    # the other tags float32
    "spearman": (FLOAT, INVALID, "spearman inputs and output must be floating point (dtype tags %d, 0, 0)",
                 lambda L, b, d: L.mb200_spearman_corrcoef(b.p, d, b.t, F32, N, 1, b.out, F32, 1e-6, b.ws, NBYTES, b.err, 0)),
    "kendall": (FLOAT | {_native.I32, I64}, INVALID, "kendall inputs must be floating point, int32 or int64 (dtype tags %d, 0)",
                lambda L, b, d: L.mb200_kendall_rank_corrcoef(b.p, d, b.t, F32, N, 1, 1, 0, b.out, F32, None, b.ws, NBYTES, b.err, 0)),
    "kendall_target": (FLOAT | {_native.I32, I64}, INVALID, "kendall inputs must be floating point, int32 or int64 (dtype tags 0, %d)",
                       lambda L, b, d: L.mb200_kendall_rank_corrcoef(b.p, F32, b.t, d, N, 1, 1, 0, b.out, F32, None, b.ws, NBYTES,
                                                                     b.err, 0)),
    # int64 target: two images of 8 points, 2 categories, the smallest tables
    "panoptic_update": (LABELS - {_native.BOOL}, INVALID, "bad sizes, capacities or dtype tags (%d, 4)",
                        lambda L, b, d: L.mb200_panoptic_update(b.p, d, b.t, I64, 2, 8, b.cats, 2, 1, 0, 0, 2, 64, 64, b.iou, b.tp,
                                                                b.fp, b.fn, b.ws, NBYTES, b.err, 0)),
    "hausdorff_one_hot": (LABELS, INVALID, "unsupported dtype tags %d, 4", lambda L, b, d: _hausdorff(L, b, d, 1)),
    "hausdorff_index": ({I64}, INVALID, "index labels must be int64 (dtype tags %d, 4)", lambda L, b, d: _hausdorff(L, b, d, 0)),
}

# K20 and K21 on one 16 x 16 (SSIM) or 48 x 48 (VIF, UQI) image: call(lib, buffers, preds tag, target tag)
SSIM_GEO = (1, 1, 1, 16, 16) + (256, 256, 0, 16, 1) * 2
VIF_GEO = (1, 1, 1, 48, 48) + (2304, 2304, 0, 48, 1) * 2
_IMAGE = {
    "ssim_update": lambda L, b, dp, dt: L.mb200_ssim_update(b.p, dp, b.t, dt, *SSIM_GEO, 1, 3, 3, 0, 1, 1, 0, b.weights, 0, 0.0, 0.0,
                                                            None, 1.0, 1.0, b.out, None, None, b.ws, NBYTES, 0),
    "ssim_data_range": lambda L, b, dp, dt: L.mb200_ssim_data_range(b.p, dp, b.t, dt, *SSIM_GEO, 0.01, 0.03, b.acc, b.ws, NBYTES, 0),
    "ssim_avg_pool": lambda L, b, dp, dt: L.mb200_ssim_avg_pool(b.p, dp, b.t, dt, *SSIM_GEO, 0, b.out, b.acc, 0),
    "vif_scale_update": lambda L, b, dp, dt: L.mb200_vif_scale_update(b.p, dp, b.t, dt, *VIF_GEO, 1, 17, 17, b.weights, 1e-10, 2.0,
                                                                      b.fps, b.tps, b.ws, NBYTES, 0),
    "vif_decimate": lambda L, b, dp, dt: L.mb200_vif_decimate(b.p, dp, b.t, dt, *VIF_GEO, 9, 9, b.weights, b.out, b.acc, 0),
    "uqi_update": lambda L, b, dp, dt: L.mb200_uqi_update(b.p, dp, b.t, dt, *VIF_GEO, 1, 11, 11, 0, 5, 5, 5, 5, b.weights, 1e-7,
                                                          b.out, None, b.ws, NBYTES, 0),
}
for _name, _call in _IMAGE.items():
    # the preds tag varied with a float32 target, then the target tag with float32 preds
    ENTRIES[_name] = (FLOAT, INVALID, "preds must be a floating-point tensor (dtype tag %d)",
                      lambda L, b, d, _call=_call: _call(L, b, d, F32))
    ENTRIES[_name + "_target"] = (FLOAT, INVALID, "target must be a floating-point tensor (dtype tag %d)",
                                  lambda L, b, d, _call=_call: _call(L, b, F32, d))


@pytest.mark.parametrize("name", sorted(ENTRIES))
def test_rejected_tags_fail_before_any_cuda_work(name):
    accepted, code, msg, call = ENTRIES[name]
    if code is None:
        pytest.skip("the entry point rejects no tag")
    lib = _native.lib()
    for d in TAGS:
        if d in accepted:
            continue
        launches = lib.mb200_launch_count()
        rc = call(lib, _BUF, d)
        assert rc == code, (name, d, rc, lib.mb200_last_error())
        assert lib.mb200_last_error().decode() == msg % d, (name, d)
        assert lib.mb200_launch_count() == launches, (name, d)


@pytest.mark.parametrize("name", sorted(ENTRIES))
def test_accepted_tags_reach_the_first_cuda_call(name):
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present: accepted tags would launch kernels on these buffers")
    accepted, _, _, call = ENTRIES[name]
    lib = _native.lib()
    for d in sorted(accepted):
        rc = call(lib, _BUF, d)
        assert rc == -2 and lib.mb200_last_error().startswith(b"CUDA error"), (name, d, rc, lib.mb200_last_error())
