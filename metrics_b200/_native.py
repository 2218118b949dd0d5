"""ctypes binding of the C-ABI in ``include/metrics_b200.h`` (``_lib/libmetrics_b200.so``).

This is the only place where Python crosses into the hand-written sm_90a kernels.  There is deliberately NO
CPU or PyTorch fallback: if the shared library is missing, or a tensor handed to a kernel wrapper does not
live on a CUDA device, we raise immediately.
"""
from __future__ import annotations

import ctypes
import os
import weakref
from typing import Optional

import torch
from torch import Tensor

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_lib", "libmetrics_b200.so")
_lib: Optional[ctypes.CDLL] = None

# enum mb200_dtype
F32, F16, BF16, F64, I64, I32, I16, I8, U8, BOOL = range(10)
_DTYPE_TAG = {
    torch.float32: F32,
    torch.float16: F16,
    torch.bfloat16: BF16,
    torch.float64: F64,
    torch.int64: I64,
    torch.int32: I32,
    torch.int16: I16,
    torch.int8: I8,
    torch.uint8: U8,
    torch.bool: BOOL,
}

ABI_VERSION = 1  # MB200_ABI_VERSION of include/metrics_b200.h
# second binding of the same C-ABI: the registered PyTorch operators (metrics_b200/torch_ops.py) instead of ctypes
_TORCH_BINDING = os.environ.get("MB200_BINDING", "ctypes") == "torch"


def _ops():
    from metrics_b200 import torch_ops

    return torch_ops.ops()
FLAG_TARGET_RANGE = 1
FLAG_PREDS_RANGE = 2
FLAG_SPIN_TIMEOUT = 4
FLAG_CAPACITY = 8


class NativeLibraryError(RuntimeError):
    """The CUDA extension is missing or a kernel call failed."""


def lib_path() -> str:
    return _LIB_PATH


def lib() -> ctypes.CDLL:
    """Load (once) and return the shared library; fail loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise NativeLibraryError(
                f"metrics_b200: CUDA extension not built: {_LIB_PATH} is missing. Run "
                "`python -c 'import __graft_entry__ as g; g.build()'` (or `make -C metrics_b200/csrc`). "
                "There is no CPU fallback."
            )
        handle = ctypes.CDLL(_LIB_PATH)
        declare_signatures(handle)
        if handle.mb200_abi_version() != ABI_VERSION:
            raise NativeLibraryError(
                f"metrics_b200: {_LIB_PATH} implements C-ABI version {handle.mb200_abi_version()}, this package binds version "
                f"{ABI_VERSION} (include/metrics_b200.h): rebuild it with `python -c 'import __graft_entry__ as g; g.build()'`."
            )
        _lib = handle
    return _lib


# Return / argument types of every entry point of include/metrics_b200*.h, one letter per C type (tests/test_abi.py
# re-derives this table from the headers and fails when they drift apart).  Declaring them lets ctypes convert plain Python
# ints / floats / None itself — no `c_void_p` / `c_int64` object per argument on the launch path, a large share of the host
# time of a small `update()` — and makes a wrong argument count or kind a TypeError instead of a silent truncation.
_C_TYPES = {"i": ctypes.c_int, "q": ctypes.c_int64, "Q": ctypes.c_uint64, "d": ctypes.c_double, "p": ctypes.c_void_p,
            "s": ctypes.c_char_p}
_VOL = "pipi" + "q" * 15  # image kernels: preds, its tag, target, its tag, [b, c, d, h, w], preds strides, target strides
SIGNATURES = {
    # include/metrics_b200.h
    "mb200_abi_version": ("i", ""),
    "mb200_last_error": ("s", ""),
    "mb200_launch_count": ("Q", ""),
    "mb200_multiclass_confmat_update": ("i", "piipiqqqiqppp"),
    "mb200_multiclass_stat_scores_update": ("i", "piipiqqqiqippppppp"),
    "mb200_multiclass_stat_scores_topk_update": ("i", "pipiqqqiqppppppp"),
    "mb200_multiclass_stat_scores_samplewise": ("i", "piipiqqqiqpppp"),
    "mb200_argmax_rows": ("i", "piqqqpp"),
    "mb200_curve_sigmoid_if_logits": ("i", "piqppp"),
    "mb200_curve_softmax_if_logits": ("i", "piqqppp"),
    "mb200_curve_normalize_scratch_bytes": ("q", "q"),
    "mb200_curve_sigmoid_if_logits_scratch": ("i", "piqppqp"),
    "mb200_curve_softmax_if_logits_scratch": ("i", "piqqppqp"),
    "mb200_curve_workspace_bytes": ("q", "qq"),
    "mb200_curve_workspace_bytes_for": ("q", "qqi"),
    "mb200_curve_weighted_workspace_bytes": ("q", "qi"),
    "mb200_curve_weighted_clf_curve": ("i", "pipipqqpqpppppp"),
    "mb200_curve_pack_keys": ("i", "piqqpp"),
    "mb200_curve_evaluate_keys": ("i", "ppiqqqpqppppp"),
    "mb200_curve_evaluate_keys_nonneg": ("i", "ppiqqqpqppppp"),
    "mb200_curve_evaluate": ("i", "pipiqqqpqpppppppp"),
    "mb200_curve_evaluate_nonneg": ("i", "pipiqqqpqpppppppp"),
    "mb200_curve_evaluate_multilabel": ("i", "pipiqqiqpqpppppppp"),
    "mb200_coco_map_workspace_bytes": ("q", "qqq"),
    "mb200_coco_map_evaluate": ("i", "pppppppppqqqqqpqipqpqpqpqppppp"),
    "mb200_coco_map_match": ("i", "pppppppppqqqpqpqqppppppp"),
    "mb200_coco_map_match_ex": ("i", "pppppppppqqqpqipqqppppippppppp"),
    "mb200_mask_pack_bits": ("i", "pqqpqpp"),
    "mb200_mask_pack_entry": ("i", "pqqqpp"),
    "mb200_kl_divergence_rows": ("i", "ppiqqipp"),
    "mb200_mask_pair_intersections": ("i", "pppppppppipqqpp"),
    "mb200_coco_map_accumulate": ("i", "pppppqpqqqqpqpqpqppppp"),
    "mb200_binary_stat_counts": ("i", "pipiqqqdiqipppp"),
    "mb200_binary_stat_counts_scratch": ("i", "pipiqqqdiqippqpp"),
    "mb200_regression_num_sums": ("i", "i"),
    "mb200_regression_scratch_doubles": ("q", "qqi"),
    "mb200_regression_sums": ("i", "ppiqqiddppp"),
    "mb200_binned_curve_scratch_words": ("q", "qq"),
    "mb200_binned_curve_compare_dtype": ("i", "iiqqi"),
    "mb200_binned_curve_update": ("i", "pipiqqpiiqppp"),
    "mb200_binned_curve_update_multilabel": ("i", "pipiqqpiiqiqppp"),
    "mb200_multiclass_stats_softmax_update": ("i", "pipiqqippppppppp"),
    "mb200_peer_pack_keys_put": ("i", "piqqqiqqpqp"),
    "mb200_peer_put_all": ("i", "pqpqip"),
    "mb200_peer_reduce_put_i64": ("i", "pqqqiiip"),
    # include/metrics_b200_calibration.h
    "mb200_calibration_scratch_bytes": ("q", "q"),
    "mb200_calibration_top_label": ("i", "pipiqqiqpppqpp"),
    "mb200_calibration_bin_scratch_bytes": ("q", "qq"),
    "mb200_calibration_bin_sums": ("i", "pipiqpqppppqp"),
    # include/metrics_b200_segmentation.h
    "mb200_segmentation_scratch_bytes": ("q", "qqqiiii"),
    "mb200_segmentation_overlap_counts": ("i", "pipiqqqiiqqiippqpp"),
    # include/metrics_b200_retrieval.h
    "mb200_retrieval_index_range": ("i", "pqpp"),
    "mb200_retrieval_sort_scratch_bytes": ("q", "qi"),
    "mb200_retrieval_sort": ("i", "pppiqqqpppppqp"),
    "mb200_retrieval_ideal_scratch_bytes": ("q", "qi"),
    "mb200_retrieval_sort_ideal": ("i", "ppqippqpp"),
    "mb200_retrieval_evaluate_scratch_bytes": ("q", "q"),
    "mb200_retrieval_evaluate": ("i", "pppppqiqipppqp"),
    "mb200_retrieval_auroc": ("i", "ppppqqdpppqp"),
    "mb200_retrieval_pr_curve_scratch_bytes": ("q", "q"),
    "mb200_retrieval_pr_curve": ("i", "ppppqqippppqp"),
    # include/metrics_b200_rankcorr.h
    "mb200_rankcorr_scratch_bytes": ("q", "qqi"),
    "mb200_spearman_corrcoef": ("i", "pipiqqpidpqpp"),
    "mb200_kendall_rank_corrcoef": ("i", "pipiqqiipippqpp"),
    # include/metrics_b200_panoptic.h
    "mb200_panoptic_scratch_bytes": ("q", "qqqqqqii"),
    "mb200_panoptic_update": ("i", "pipiqqpqqiiqqqpppppqpp"),
    # include/metrics_b200_hausdorff.h
    "mb200_hausdorff_scratch_bytes": ("q", "qqiq"),
    "mb200_hausdorff_distance": ("i", "pipiiqqqqqqqqqqqqiiiddiqppqpp"),
    # include/metrics_b200_image.h
    "mb200_ssim_scratch_bytes": ("q", "iqqqqqiiiiii"),
    "mb200_ssim_data_range": ("i", _VOL + "ddppqp"),
    "mb200_ssim_update": ("i", _VOL + "iiiiiiipiddpddppppqp"),
    "mb200_ssim_avg_pool": ("i", _VOL + "ippp"),
    "mb200_vif_scale_update": ("i", _VOL + "iiipddpppqp"),
    "mb200_vif_decimate": ("i", _VOL + "iipppp"),
    "mb200_uqi_update": ("i", _VOL + "iiiiiiiipdpppqp"),
}


def declare_signatures(handle) -> None:
    """Set ``restype`` / ``argtypes`` of every exported function on a loaded library handle."""
    for name, (ret, args) in SIGNATURES.items():
        fn = getattr(handle, name)
        fn.restype = _C_TYPES[ret]
        fn.argtypes = [_C_TYPES[a] for a in args]


def launch_count() -> int:
    return int(lib().mb200_launch_count())


def tag(t: Tensor) -> int:
    try:
        return _DTYPE_TAG[t.dtype]
    except KeyError:
        raise TypeError(f"metrics_b200: unsupported tensor dtype {t.dtype}") from None


def require_cuda(*tensors: Tensor) -> torch.device:
    """All tensors must live on the same CUDA device (the kernels have no host implementation)."""
    dev = None
    for t in tensors:
        if not t.is_cuda:
            raise NativeLibraryError(
                "metrics_b200 kernels only run on CUDA tensors (sm_90a); got a tensor on "
                f"'{t.device}'. Move the metric and its inputs to the GPU: there is no CPU fallback."
            )
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise RuntimeError(
                f"Expected all tensors to be on the same device, but found at least two devices, {dev} and {t.device}!"
            )
    return dev


class _NoOp:
    def __enter__(self) -> None:
        return None

    def __exit__(self, *exc: object) -> None:
        return None


_NOOP = _NoOp()


def on_device(device: torch.device):
    """Context that makes ``device`` current for the launch; free when it already is (the common case)."""
    if torch.cuda.current_device() == device.index:
        return _NOOP
    return torch.cuda.device(device)


def ptr(t: Optional[Tensor]) -> Optional[int]:
    """Device address for a ``void*`` parameter (``None`` -> NULL); ctypes converts it, see `declare_signatures`."""
    return None if t is None else t.data_ptr()


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def stream_handle(device: torch.device) -> int:
    """``cudaStream_t`` of torch's current stream on ``device`` as an integer (raw-pointer query: no Stream object per
    launch; 0 is the legacy default stream)."""
    if _raw_stream is not None:
        return _raw_stream(device.index if device.index is not None else torch.cuda.current_device())
    return torch.cuda.current_stream(device).cuda_stream


_flag_words: dict = {}


def _flag_scratch(device: torch.device, stream: int) -> Tensor:
    """4-byte device word for the batch-global "are these logits?" vote, one per (device, stream): launches on one stream
    are ordered, so consecutive format calls can share it; different streams never do."""
    key = (device.index, stream)
    t = _flag_words.get(key)
    if t is None:
        t = torch.zeros(1, dtype=torch.int32, device=device)
        _flag_words[key] = t
    return t


def i64(v: int) -> int:
    """Value for an ``int64_t`` parameter."""
    return int(v)


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().mb200_last_error().decode("utf-8", "replace")
        if rc == -1:
            raise ValueError(f"metrics_b200.{what}: {msg}")
        raise NativeLibraryError(f"metrics_b200.{what} failed (code {rc}): {msg}")


# ----------------------------------------------------------------------------------------------------------
# K1 wrappers
# ----------------------------------------------------------------------------------------------------------
def _class_dim_geometry(preds: Tensor, has_class_dim: bool) -> tuple[int, int]:
    """(n_outer, inner) of a contiguous [N, C, ...] (or label [N, ...]) tensor."""
    if has_class_dim:
        n_outer = preds.shape[0]
        inner = 1
        for s in preds.shape[2:]:
            inner *= s
        return n_outer, inner
    return preds.numel(), 1


def multiclass_confmat_update_(
    confmat: Tensor,
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    ignore_index: Optional[int],
    err_flag: Optional[Tensor] = None,
) -> None:
    """In-place ``confmat[t, argmax(preds)] += 1`` (``mb200_multiclass_confmat_update``).  Launch path of cfg1 / cfg2:
    arguments are handed to ctypes as plain ints (see `declare_signatures`), no helper call per argument."""
    if _TORCH_BINDING:
        _ops().confmat_update_(confmat, preds, target, int(num_classes), ignore_index, err_flag)
        return
    dev = require_cuda(confmat, preds, target)
    has_class_dim = preds.ndim == target.ndim + 1
    preds = preds.contiguous()
    target = target.contiguous()
    n_outer, inner = _class_dim_geometry(preds, has_class_dim)
    with on_device(dev):
        rc = lib().mb200_multiclass_confmat_update(
            preds.data_ptr(), tag(preds), has_class_dim, target.data_ptr(), tag(target), n_outer, int(num_classes), inner,
            ignore_index is not None, int(ignore_index or 0), confmat.data_ptr(),
            None if err_flag is None else err_flag.data_ptr(), stream_handle(dev),
        )
    if rc:
        check(rc, "multiclass_confmat_update")


def multiclass_stat_scores_update_(
    tp: Tensor,
    fp: Tensor,
    tn: Tensor,
    fn: Tensor,
    workspace: Tensor,
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    ignore_index: Optional[int],
    micro: bool,
    err_flag: Optional[Tensor] = None,
) -> None:
    """In-place tp/fp/tn/fn accumulation (``mb200_multiclass_stat_scores_update``).  The four states and the workspace
    belong to one metric and move together (`Metric._apply`), so one of them stands for all in the device check."""
    if _TORCH_BINDING:
        _ops().stat_scores_update_(tp, fp, tn, fn, workspace, preds, target, int(num_classes), ignore_index, bool(micro), err_flag)
        return
    dev = require_cuda(tp, workspace, preds, target)
    has_class_dim = preds.ndim == target.ndim + 1
    preds = preds.contiguous()
    target = target.contiguous()
    n_outer, inner = _class_dim_geometry(preds, has_class_dim)
    with on_device(dev):
        rc = lib().mb200_multiclass_stat_scores_update(
            preds.data_ptr(), tag(preds), has_class_dim, target.data_ptr(), tag(target), n_outer, int(num_classes), inner,
            ignore_index is not None, int(ignore_index or 0), bool(micro), tp.data_ptr(), fp.data_ptr(), tn.data_ptr(),
            fn.data_ptr(), workspace.data_ptr(), None if err_flag is None else err_flag.data_ptr(), stream_handle(dev),
        )
    if rc:
        check(rc, "multiclass_stat_scores_update")


def multiclass_stats_softmax_update_(tp: Tensor, fp: Tensor, tn: Tensor, fn: Tensor, workspace: Tensor, preds: Tensor,
                                     target: Tensor, num_classes: int, micro: bool, err_flag: Optional[Tensor] = None) -> Tensor:
    """K11 (``mb200_multiclass_stats_softmax_update``): in-place tp/fp/tn/fn accumulation AND the batch's
    ``normalize_logits_if_needed(preds, "softmax")`` from one read of ``preds [N, C]``; returns the probabilities."""
    if _TORCH_BINDING:
        return _ops().stats_softmax_update_(tp, fp, tn, fn, workspace, preds, target, int(num_classes), bool(micro), err_flag)
    dev = require_cuda(tp, workspace, preds, target)
    preds = preds.contiguous()
    target = target.contiguous()
    probs = torch.empty_like(preds)
    st = stream_handle(dev)
    with on_device(dev):
        rc = lib().mb200_multiclass_stats_softmax_update(
            preds.data_ptr(), tag(preds), target.data_ptr(), tag(target), preds.shape[0], int(num_classes), bool(micro),
            tp.data_ptr(), fp.data_ptr(), tn.data_ptr(), fn.data_ptr(), workspace.data_ptr(), probs.data_ptr(),
            _flag_scratch(dev, st).data_ptr(), None if err_flag is None else err_flag.data_ptr(), st,
        )
    if rc:
        check(rc, "multiclass_stats_softmax_update")
    return probs


def argmax_rows(preds: Tensor) -> Tensor:
    """``preds.argmax(dim=1)`` for a floating [N, C, ...] tensor, torch tie/NaN semantics."""
    dev = require_cuda(preds)
    preds = preds.contiguous()
    n_outer, inner = _class_dim_geometry(preds, True)
    out = torch.empty((preds.shape[0], *preds.shape[2:]), dtype=torch.int64, device=dev)
    with on_device(dev):
        rc = lib().mb200_argmax_rows(
            ptr(preds), tag(preds), i64(n_outer), i64(preds.shape[1]), i64(inner), ptr(out), stream_handle(dev)
        )
    check(rc, "argmax_rows")
    return out


# ----------------------------------------------------------------------------------------------------------
# K3/K5/K6 wrappers (exact curve family)
# ----------------------------------------------------------------------------------------------------------
def sigmoid_if_logits(preds: Tensor) -> Tensor:
    """``normalize_logits_if_needed(preds, "sigmoid")``: per-call global range test + conditional sigmoid, no host sync."""
    if _TORCH_BINDING:
        return _ops().normalize_logits_if_needed(preds, "sigmoid")
    dev = require_cuda(preds)
    preds = preds.contiguous()
    out = torch.empty_like(preds)
    if preds.numel() == 0:
        return out
    st = stream_handle(dev)
    n = preds.numel()
    with on_device(dev):
        if n <= 32768:  # one-CTA kernel: the shared per-stream vote word is all it needs
            rc = lib().mb200_curve_sigmoid_if_logits(preds.data_ptr(), tag(preds), n, out.data_ptr(),
                                                     _flag_scratch(dev, st).data_ptr(), st)
        else:  # large batches: speculative single pass, needs one byte of scratch per 16 KB tile
            nbytes = int(lib().mb200_curve_normalize_scratch_bytes(n))
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            rc = lib().mb200_curve_sigmoid_if_logits_scratch(preds.data_ptr(), tag(preds), n, out.data_ptr(),
                                                             scratch.data_ptr(), nbytes, st)
    if rc != 0:
        check(rc, "curve_sigmoid_if_logits")
    return out


def softmax_if_logits(preds: Tensor) -> Tensor:
    """``normalize_logits_if_needed(preds, "softmax")`` for a contiguous ``[N, C]`` tensor."""
    if _TORCH_BINDING:
        return _ops().normalize_logits_if_needed(preds, "softmax")
    dev = require_cuda(preds)
    preds = preds.contiguous()
    out = torch.empty_like(preds)
    if preds.numel() == 0:
        return out
    st = stream_handle(dev)
    n, c = preds.shape[0], preds.shape[1]
    with on_device(dev):
        if c <= 1024 and preds.dtype != torch.float64:  # speculative single pass: one pending byte per row behind the vote word
            scratch = torch.empty(8 + n, dtype=torch.uint8, device=dev)
            rc = lib().mb200_curve_softmax_if_logits_scratch(preds.data_ptr(), tag(preds), n, c, out.data_ptr(),
                                                             scratch.data_ptr(), 8 + n, st)
        else:
            rc = lib().mb200_curve_softmax_if_logits(ptr(preds), tag(preds), i64(n), i64(c), ptr(out), ptr(_flag_scratch(dev, st)), st)
    check(rc, "curve_softmax_if_logits")
    return out


def curve_evaluate(preds: Tensor, target: Tensor, num_classes: int = 1, pos_label: int = 1, want_curve: bool = False,
                   unit_range: Optional[bool] = None):
    """Sort + TP/FP scan for ``num_classes`` one-vs-rest curves (``mb200_curve_evaluate`` / ``mb200_curve_evaluate_nonneg``).

    Returns ``(auroc[C] f32, ap[C] f32, counts[C, 3] i64, curve)`` where ``curve`` is ``None`` or the tuple
    ``(fps, tps, thresholds)`` of ``[C, N]`` buffers whose first ``counts[c, 2]`` entries per row are valid; fps / tps are
    float32, thresholds float64 for float64 scores (sorted as 64-bit keys) and float32 otherwise.

    ``unit_range``: non-negative (or NaN) scores — anything in [0, 1] — sort as 4-byte keys with the label in bit 0 (the
    ``_nonneg`` entry).  ``True`` is the
    caller's promise (metric states: ``normalize_logits_if_needed`` ran on them) and is not checked here; ``None`` tries that
    path, reads the kernel's range flag back (one host sync — every caller reads ``counts`` on the host next anyway) and
    re-evaluates on the general path if a score was outside; ``False`` takes the general path.
    """
    if _TORCH_BINDING:
        auroc, ap, counts, fps, tps, thr = _ops().curve_evaluate(preds, target, int(num_classes), int(pos_label), bool(want_curve))
        return auroc, ap, counts, ((fps, tps, thr) if want_curve else None)
    dev = require_cuda(preds, target)
    preds = preds.contiguous()
    target = target.contiguous()
    n = target.numel()
    lib_ = lib()
    nbytes = int(lib_.mb200_curve_workspace_bytes_for(i64(num_classes), i64(n), tag(preds)))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    auroc = torch.empty(num_classes, dtype=torch.float32, device=dev)
    ap = torch.empty(num_classes, dtype=torch.float32, device=dev)
    counts = torch.empty((num_classes, 3), dtype=torch.int64, device=dev)
    curve = None
    if want_curve:
        thr_dtype = torch.float64 if preds.dtype == torch.float64 else torch.float32
        curve = tuple(torch.empty((num_classes, n), dtype=dt, device=dev) for dt in (torch.float32, torch.float32, thr_dtype))
    unit = unit_range is not False and preds.dtype != torch.float64 and n > 0
    flag = torch.zeros(1, dtype=torch.int32, device=dev) if unit and unit_range is None else None
    with on_device(dev):
        for entry in ((lib_.mb200_curve_evaluate_nonneg, lib_.mb200_curve_evaluate) if unit else (lib_.mb200_curve_evaluate,)):
            rc = entry(
                ptr(preds), tag(preds), ptr(target), tag(target), i64(n), i64(num_classes), i64(pos_label), ptr(ws),
                i64(nbytes), ptr(auroc), ptr(ap), ptr(counts), ptr(curve[0] if curve else None),
                ptr(curve[1] if curve else None), ptr(curve[2] if curve else None), ptr(flag), stream_handle(dev),
            )
            check(rc, "curve_evaluate")
            if flag is None or int(flag) == 0:
                break
            flag = None  # a negative score: once more on the general path
    return auroc, ap, counts, curve


def curve_weighted_clf_curve(preds: Tensor, target: Tensor, weights: Tensor, pos_label: int = 1):
    """``(fps f64 [U], tps f64 [U], thresholds [U])`` of the weighted binary curve (``mb200_curve_weighted_clf_curve``); U is
    read back from the device (data-dependent output size, like the reference's ``torch.where``)."""
    dev = require_cuda(preds, target, weights)
    preds, target = preds.contiguous(), target.contiguous()
    weights = weights.to(torch.float64).contiguous()
    n = preds.numel()
    lib_ = lib()
    nbytes = int(lib_.mb200_curve_weighted_workspace_bytes(n, tag(preds)))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    fps = torch.empty(n, dtype=torch.float64, device=dev)
    tps = torch.empty(n, dtype=torch.float64, device=dev)
    thr = torch.empty(n, dtype=torch.float64 if preds.dtype == torch.float64 else torch.float32, device=dev)
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    with on_device(dev):
        rc = lib_.mb200_curve_weighted_clf_curve(ptr(preds), tag(preds), ptr(target), tag(target), ptr(weights), n,
                                                 int(pos_label), ptr(ws), nbytes, ptr(fps), ptr(tps), ptr(thr), ptr(count),
                                                 None, stream_handle(dev))
    check(rc, "curve_weighted_clf_curve")
    u = int(count.item())
    return fps[:u], tps[:u], thr[:u]


# ----------------------------------------------------------------------------------------------------------
# K8 wrapper (COCO mAP)
# ----------------------------------------------------------------------------------------------------------
def coco_map_evaluate(
    det_box: Tensor, det_score: Tensor, det_label: Tensor, det_counts: list,
    gt_box: Tensor, gt_label: Tensor, gt_crowd: Tensor, gt_area: Tensor, gt_counts: list,
    classes: Tensor, micro: bool, iou_thresholds: list, rec_thresholds: list, max_dets: list,
):
    """``mb200_coco_map_evaluate``: returns ``precision [T,R,K,A,M]``, ``recall [T,K,A,M]``, ``scores`` (float64)."""
    import numpy as np

    dev = require_cuda(det_box, det_score, det_label, gt_box, gt_label, gt_crowd, gt_area, classes)
    n_img = len(det_counts)
    det_off = torch.from_numpy(np.concatenate([[0], np.cumsum(det_counts)]).astype(np.int32)).to(dev, non_blocking=True)
    gt_off = torch.from_numpy(np.concatenate([[0], np.cumsum(gt_counts)]).astype(np.int32)).to(dev, non_blocking=True)
    n_det, n_gt = int(sum(det_counts)), int(sum(gt_counts))
    K = 1 if micro else int(classes.numel())
    T, R, M = len(iou_thresholds), len(rec_thresholds), len(max_dets)
    det_box = det_box.to(torch.float32).contiguous()
    det_score = det_score.to(torch.float32).contiguous()
    det_label = det_label.to(torch.int64).contiguous()
    gt_box = gt_box.to(torch.float32).contiguous()
    gt_label = gt_label.to(torch.int64).contiguous()
    gt_crowd = gt_crowd.to(torch.uint8).contiguous()
    gt_area = gt_area.to(torch.float64).contiguous()
    classes = classes.to(torch.int64).contiguous()
    rec_dev = torch.tensor(rec_thresholds, dtype=torch.float64).to(dev, non_blocking=True)
    lib_ = lib()
    nbytes = int(lib_.mb200_coco_map_workspace_bytes(i64(n_det), i64(max(1, classes.numel())), i64(M)))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    precision = torch.empty((T, R, K, 4, M), dtype=torch.float64, device=dev)
    recall = torch.empty((T, K, 4, M), dtype=torch.float64, device=dev)
    scores = torch.empty((T, R, K, 4, M), dtype=torch.float64, device=dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    iou_host = (ctypes.c_double * T)(*[float(x) for x in iou_thresholds])
    md_host = (ctypes.c_int64 * M)(*[int(x) for x in max_dets])
    with on_device(dev):
        rc = lib_.mb200_coco_map_evaluate(
            ptr(det_box), ptr(det_score), ptr(det_label), ptr(det_off), ptr(gt_box), ptr(gt_label), ptr(gt_crowd),
            ptr(gt_area), ptr(gt_off), i64(n_img), i64(n_det), i64(n_gt), i64(max(det_counts) if det_counts else 0),
            i64(max(gt_counts) if gt_counts else 0), ptr(classes), i64(max(1, classes.numel())), int(micro), iou_host,
            i64(T), ptr(rec_dev), i64(R), md_host, i64(M), ptr(ws), i64(nbytes), ptr(precision), ptr(recall),
            ptr(scores), ptr(err), stream_handle(dev),
        )
    if rc == -3:
        raise NotImplementedError("metrics_b200: " + lib_.mb200_last_error().decode("utf-8", "replace"))
    check(rc, "coco_map_evaluate")
    return precision, recall, scores, err


def mask_pack_bits(masks: Tensor):
    """``mb200_mask_pack_bits``: boolean / uint8 masks ``[n, H, W]`` -> ``(words int32 [n, ceil(H*W/32)], area int64 [n])``."""
    dev = require_cuda(masks)
    if masks.dtype not in (torch.bool, torch.uint8):
        masks = masks != 0
    masks = masks.contiguous()
    n = int(masks.shape[0])
    hw = int(masks[0].numel()) if n else 0
    words = (hw + 31) // 32
    out = torch.empty((n, words), dtype=torch.int32, device=dev)
    area = torch.empty(n, dtype=torch.int64, device=dev)
    if n:
        with on_device(dev):
            rc = lib().mb200_mask_pack_bits(masks.view(torch.uint8).data_ptr(), n, hw, out.data_ptr() if words else None, words,
                                            area.data_ptr(), stream_handle(dev))
        check(rc, "mask_pack_bits")
    return out, area


def mask_pack_entry(masks: Tensor) -> Tensor:
    """``mb200_mask_pack_entry``: boolean / uint8 masks ``[n, H, W]`` -> the int32 state entry ``[n, H, W, areas.., bit rows..]``."""
    dev = require_cuda(masks)
    if masks.dtype not in (torch.bool, torch.uint8):
        masks = masks != 0
    masks = masks.contiguous()
    n, h, w = (int(x) for x in masks.shape)
    out = torch.empty(3 + n + n * ((h * w + 31) // 32), dtype=torch.int32, device=dev)
    with on_device(dev):
        rc = lib().mb200_mask_pack_entry(masks.view(torch.uint8).data_ptr() if masks.numel() else None, n, h, w, out.data_ptr(),
                                         stream_handle(dev))
    check(rc, "mask_pack_entry")
    return out


def mask_pair_intersections(det_words: Tensor, det_word_off: Tensor, gt_words: Tensor, gt_word_off: Tensor, det_off: Tensor,
                            gt_off: Tensor, img_words: Tensor, det_label: Tensor, gt_label: Tensor, micro: bool,
                            pair_off: Tensor, n_pairs: int, max_pairs_per_img: int) -> Tensor:
    """``mb200_mask_pair_intersections``: the flat per-image ``[D_i, G_i]`` tables of intersection pixel counts (float64)."""
    dev = require_cuda(det_words, gt_words, det_word_off, gt_word_off, det_off, gt_off, img_words, det_label, gt_label, pair_off)
    out = torch.empty(max(1, n_pairs), dtype=torch.float64, device=dev)
    n_img = int(img_words.numel())
    if n_img and n_pairs:
        with on_device(dev):
            rc = lib().mb200_mask_pair_intersections(
                ptr(det_words), ptr(det_word_off), ptr(gt_words), ptr(gt_word_off), ptr(det_off), ptr(gt_off), ptr(img_words),
                ptr(det_label), ptr(gt_label), 1 if micro else 0, ptr(pair_off), n_img, int(max_pairs_per_img), ptr(out),
                stream_handle(dev))
        check(rc, "mask_pair_intersections")
    return out


def coco_map_match(det_box: Tensor, det_score: Tensor, det_label: Tensor, det_counts: list, gt_box: Tensor, gt_label: Tensor,
                   gt_crowd: Tensor, gt_area: Tensor, gt_counts: list, classes: Tensor, iou_thresholds: list, max_det_last: int,
                   micro: bool = False, masks: Optional[dict] = None, gt_area_exact: bool = False):
    """``mb200_coco_map_match`` (``_ex`` with any of the last three arguments): COCOeval.evaluateImg for the given images only.
    Returns the per-detection records ``(det_cat i32 [n], det_rank i32 [n], det_match i64 [n], det_ignore i64 [n])``, ``npig``
    i32 ``[K, 4]`` and the error word.  ``masks``: ``{"pair_inter", "pair_off", "det_area", "gt_area"}`` (float64 / int64 /
    float64 / float64 device tensors) switches the IoU from boxes to instance masks."""
    import numpy as np

    dev = require_cuda(det_box, det_score, det_label, gt_box, gt_label, gt_crowd, gt_area, classes)
    n_img = len(det_counts)
    det_off = torch.from_numpy(np.concatenate([[0], np.cumsum(det_counts)]).astype(np.int32)).to(dev, non_blocking=True)
    gt_off = torch.from_numpy(np.concatenate([[0], np.cumsum(gt_counts)]).astype(np.int32)).to(dev, non_blocking=True)
    n_det = int(sum(det_counts))
    det_box = det_box.to(torch.float32).contiguous()
    det_score = det_score.to(torch.float32).contiguous()
    det_label = det_label.to(torch.int64).contiguous()
    gt_box = gt_box.to(torch.float32).contiguous()
    gt_label = gt_label.to(torch.int64).contiguous()
    gt_crowd = gt_crowd.to(torch.uint8).contiguous()
    gt_area = gt_area.to(torch.float64).contiguous()
    classes = classes.to(torch.int64).contiguous()
    k, t = int(classes.numel()), len(iou_thresholds)
    det_cat = torch.empty(max(n_det, 1), dtype=torch.int32, device=dev)
    det_rank = torch.empty(max(n_det, 1), dtype=torch.int32, device=dev)
    det_match = torch.empty(max(n_det, 1), dtype=torch.int64, device=dev)
    det_ignore = torch.empty(max(n_det, 1), dtype=torch.int64, device=dev)
    npig = torch.zeros((1 if micro else k, 4), dtype=torch.int32, device=dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    iou_host = (ctypes.c_double * t)(*[float(x) for x in iou_thresholds])
    max_d, max_g = (max(det_counts) if det_counts else 0), (max(gt_counts) if gt_counts else 0)
    with on_device(dev):
        if micro or masks is not None or gt_area_exact:
            m = masks or {}
            keep = [m[name].contiguous() for name in ("pair_inter", "pair_off", "det_area", "gt_area")] if masks else [None] * 4
            rc = lib().mb200_coco_map_match_ex(
                ptr(det_box), ptr(det_score), ptr(det_label), ptr(det_off), ptr(gt_box), ptr(gt_label), ptr(gt_crowd),
                ptr(gt_area), ptr(gt_off), n_img, max_d, max_g, ptr(classes), k, 1 if micro else 0, iou_host, t,
                int(max_det_last), ptr(keep[0]), ptr(keep[1]), ptr(keep[2]), ptr(keep[3]), 1 if gt_area_exact else 0,
                ptr(det_cat), ptr(det_rank), ptr(det_match), ptr(det_ignore), ptr(npig), ptr(err), stream_handle(dev))
        else:
            rc = lib().mb200_coco_map_match(
                ptr(det_box), ptr(det_score), ptr(det_label), ptr(det_off), ptr(gt_box), ptr(gt_label), ptr(gt_crowd),
                ptr(gt_area), ptr(gt_off), n_img, max_d, max_g, ptr(classes), k, iou_host, t, int(max_det_last), ptr(det_cat),
                ptr(det_rank), ptr(det_match), ptr(det_ignore), ptr(npig), ptr(err), stream_handle(dev))
    if rc == -3:
        raise NotImplementedError("metrics_b200: " + lib().mb200_last_error().decode("utf-8", "replace"))
    check(rc, "coco_map_match")
    return (det_cat[:n_det], det_rank[:n_det], det_match[:n_det], det_ignore[:n_det]), npig, err


def coco_map_accumulate(det_cat: Tensor, det_score: Tensor, det_rank: Tensor, det_match: Tensor, det_ignore: Tensor, npig: Tensor,
                        num_classes: int, class_lo: int, class_hi: int, n_iou_thr: int, rec_thresholds: list, max_dets: list):
    """``mb200_coco_map_accumulate``: COCOeval.accumulate for classes ``[class_lo, class_hi)`` over the given records (ties in
    score keep the given order).  Returns full-size ``precision [T,R,K,A,M]``, ``recall [T,K,A,M]``, ``scores`` (-1 outside)."""
    dev = require_cuda(det_cat, det_score, det_rank, det_match, det_ignore, npig)
    n_det = int(det_cat.numel())
    k, t, r, m = int(num_classes), int(n_iou_thr), len(rec_thresholds), len(max_dets)
    rec_dev = torch.tensor(rec_thresholds, dtype=torch.float64).to(dev, non_blocking=True)
    lib_ = lib()
    nbytes = int(lib_.mb200_coco_map_workspace_bytes(n_det, max(1, k), m))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    precision = torch.empty((t, r, k, 4, m), dtype=torch.float64, device=dev)
    recall = torch.empty((t, k, 4, m), dtype=torch.float64, device=dev)
    scores = torch.empty((t, r, k, 4, m), dtype=torch.float64, device=dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    md_host = (ctypes.c_int64 * m)(*[int(x) for x in max_dets])
    args = [x.contiguous() for x in (det_cat.to(torch.int32), det_score.to(torch.float32), det_rank.to(torch.int32),
                                     det_match.to(torch.int64), det_ignore.to(torch.int64), npig.to(torch.int32))]
    with on_device(dev):
        rc = lib_.mb200_coco_map_accumulate(
            ptr(args[0]) if n_det else None, ptr(args[1]) if n_det else None, ptr(args[2]) if n_det else None,
            ptr(args[3]) if n_det else None, ptr(args[4]) if n_det else None, n_det, ptr(args[5]), k, int(class_lo), int(class_hi),
            t, ptr(rec_dev), r, md_host, m, ptr(ws), nbytes, ptr(precision), ptr(recall), ptr(scores), ptr(err),
            stream_handle(dev))
    check(rc, "coco_map_accumulate")
    return precision, recall, scores, err


# ----------------------------------------------------------------------------------------------------------
# K2 wrapper (binary / multilabel counts)
# ----------------------------------------------------------------------------------------------------------
def binary_stat_counts(
    preds: Tensor, target: Tensor, num_labels: int, threshold: float, ignore_index: Optional[int], samplewise: bool,
    counts: Optional[Tensor] = None, err_flag: Optional[Tensor] = None,
) -> Tensor:
    """(tp, fp, tn, fn) per group from ``[N, L, ...]`` (multilabel) or ``[N, ...]`` (binary, ``num_labels == 1`` with no
    label dim) inputs; adds into ``counts [G, 4]`` (allocated zeroed when omitted)."""
    dev = require_cuda(preds, target)
    preds = preds.contiguous()
    target = target.contiguous()
    n_outer = preds.shape[0] if preds.ndim > 0 else 1
    total = preds.numel()
    inner = total // max(1, n_outer * num_labels) if total else 1
    groups = n_outer * num_labels if samplewise else num_labels
    if counts is None:
        counts = torch.zeros((groups, 4), dtype=torch.int64, device=dev)
    # scratch for the logits vote; large enough (MB200_BINARY_SCRATCH_BYTES) for the single-pass binary kernel's two count sets
    words = 32
    scratch = torch.empty(words, dtype=torch.int32, device=dev) if preds.is_floating_point() else None
    with on_device(dev):
        rc = lib().mb200_binary_stat_counts_scratch(
            ptr(preds), tag(preds), ptr(target), tag(target), i64(n_outer), i64(num_labels), i64(max(1, inner)),
            ctypes.c_double(float(threshold)), int(ignore_index is not None), i64(ignore_index or 0), int(samplewise),
            ptr(counts), ptr(scratch), 4 * words, ptr(err_flag), stream_handle(dev),
        )
    check(rc, "binary_stat_counts")
    return counts


# ----------------------------------------------------------------------------------------------------------
# K9 wrapper (regression running sums)
# ----------------------------------------------------------------------------------------------------------
REG_MSE, REG_MAE, REG_MAPE, REG_SMAPE, REG_WMAPE, REG_MSLE, REG_LOGCOSH, REG_MINKOWSKI, REG_R2, REG_EXPVAR, REG_TWEEDIE = range(11)
_REG_NUM_SUMS = {REG_WMAPE: 2, REG_R2: 3, REG_EXPVAR: 4, REG_TWEEDIE: 4}


def regression_compute_dtype(preds: Tensor, target: Tensor) -> torch.dtype:
    """The dtype the regression terms are computed in: the promoted dtype of the two inputs, as in the reference's
    ``preds - target``; float32 when neither input is floating point."""
    dtype = torch.promote_types(preds.dtype, target.dtype)
    return dtype if dtype.is_floating_point else torch.float32


def regression_sums(preds: Tensor, target: Tensor, op: int, num_outputs: int = 1, param: float = 0.0, eps: float = 0.0) -> Tensor:
    """``float64 [num_sums, num_outputs]`` sums of the per-element terms of regression op ``op`` (``mb200_regression_sums``)
    over the ``[numel / num_outputs, num_outputs]`` row-major view of the inputs.  The terms are computed in
    `regression_compute_dtype`; only an input of another dtype is cast."""
    dev = require_cuda(preds, target)
    d = int(num_outputs)
    if d < 1 or preds.numel() % d:
        raise ValueError(f"regression_sums: {preds.numel()} elements do not split into rows of num_outputs={d}")
    dtype = regression_compute_dtype(preds, target)
    if preds.dtype != dtype:
        preds = preds.to(dtype)
    if target.dtype != dtype:
        target = target.to(dtype)
    if _TORCH_BINDING:
        return _ops().regression_sums(preds, target, int(op), d, float(param), float(eps))
    preds = preds.contiguous()
    target = target.contiguous()
    n = preds.numel() // d
    k = _REG_NUM_SUMS.get(op, 1)
    out = torch.empty((k, d), dtype=torch.float64, device=dev)
    lib_ = lib()
    scratch = torch.empty(int(lib_.mb200_regression_scratch_doubles(i64(n), i64(d), int(op))), dtype=torch.float64, device=dev)
    with on_device(dev):
        rc = lib_.mb200_regression_sums(
            ptr(preds), ptr(target), tag(preds), i64(n), i64(d), int(op), ctypes.c_double(float(param)),
            ctypes.c_double(float(eps)), ptr(out), ptr(scratch), stream_handle(dev),
        )
    check(rc, "regression_sums")
    return out


def kl_divergence_rows(p: Tensor, q: Tensor, log_prob: bool) -> Tensor:
    """``measures [N]`` = KL(p_i || q_i) per row of the ``[N, d]`` distributions (``mb200_kl_divergence_rows``), in p's dtype."""
    dev = require_cuda(p, q)
    if not p.is_floating_point():
        p = p.float()
    if q.dtype != p.dtype:
        q = q.to(p.dtype)
    p, q = p.contiguous(), q.contiguous()
    n, d = int(p.shape[0]), int(p.shape[1])
    out = torch.empty(n, dtype=p.dtype, device=dev)
    if n:
        with on_device(dev):
            rc = lib().mb200_kl_divergence_rows(ptr(p) if d else None, ptr(q) if d else None, tag(p), i64(n), i64(d),
                                                1 if log_prob else 0, ptr(out), stream_handle(dev))
        check(rc, "kl_divergence_rows")
    return out


# ----------------------------------------------------------------------------------------------------------
# K4 wrapper (binned curve update)
# ----------------------------------------------------------------------------------------------------------
_sorted_cache: dict = {}


def _is_sorted(thr: Tensor) -> bool:
    """Is the threshold tensor ascending?  Reading the answer is a host sync, and a metric hands the SAME buffer to every
    update: remember it per tensor object and version counter.  (Not per storage address: a freed buffer's address is
    handed to the next tensor of the same size, and two views can start at the same address with different contents.)"""
    entry = _sorted_cache.get(id(thr))
    if entry is not None and entry[0]() is thr and entry[1] == thr._version:
        return entry[2]
    hit = bool((thr[1:] >= thr[:-1]).all())
    if len(_sorted_cache) > 256:
        _sorted_cache.clear()
    _sorted_cache[id(thr)] = (weakref.ref(thr), thr._version, hit)
    return hit


def binned_curve_update(preds: Tensor, target: Tensor, thresholds: Tensor, num_classes: int = 1,
                        multilabel: bool = False, ignore_index: Optional[int] = None) -> Tensor:
    """Multi-threshold confusion matrix of one batch: int64 ``[T, 2, 2]`` (``num_classes == 1``) or ``[T, C, 2, 2]``.
    ``thresholds`` may be in any order (rows of the result follow it) and of any float or integer dtype: the kernel works on
    a copy sorted in that dtype and compares ``score >= threshold`` in the dtype the reference would for this batch
    (``mb200_binned_curve_compare_dtype``: the score dtype above its size rule, the promoted dtype below it).
    ``multilabel``: ``target`` is ``[N, C]`` like ``preds``; entries that are neither 0 nor 1, or equal ``ignore_index`` in
    the target's dtype, are skipped."""
    dev = require_cuda(preds, target, thresholds)
    preds = preds.contiguous()
    target = target.contiguous()
    thr = thresholds
    order = None
    if thr.numel() > 1 and not _is_sorted(thr):
        thr, order = torch.sort(thr)
    thr = thr.contiguous()
    n = preds.shape[0] if multilabel else target.numel()
    t_count = thr.numel()
    confmat = torch.zeros((t_count, num_classes, 2, 2), dtype=torch.int64, device=dev)
    lib_ = lib()
    scratch = torch.zeros(int(lib_.mb200_binned_curve_scratch_words(i64(num_classes), i64(t_count))), dtype=torch.int64, device=dev)
    cmp = lib_.mb200_binned_curve_compare_dtype(tag(preds), tag(thr), n, num_classes, 1 if multilabel else 0)
    with on_device(dev):
        if multilabel:
            rc = lib_.mb200_binned_curve_update_multilabel(
                ptr(preds), tag(preds), ptr(target), tag(target), i64(n), i64(num_classes), ptr(thr), tag(thr), cmp, i64(t_count),
                0 if ignore_index is None else 1, 0 if ignore_index is None else int(ignore_index), ptr(confmat), ptr(scratch),
                stream_handle(dev))
        else:
            rc = lib_.mb200_binned_curve_update(
                ptr(preds), tag(preds), ptr(target), tag(target), i64(n), i64(num_classes), ptr(thr), tag(thr), cmp, i64(t_count),
                ptr(confmat), ptr(scratch), stream_handle(dev))
    check(rc, "binned_curve_update")
    if order is not None:
        inv = torch.empty_like(order)
        inv[order] = torch.arange(t_count, device=dev)
        confmat = confmat[inv]
    return confmat[:, 0] if num_classes == 1 and not multilabel else confmat


def multiclass_stat_scores_topk_update_(
    tp: Tensor, fp: Tensor, tn: Tensor, fn: Tensor, workspace: Tensor, preds: Tensor, target: Tensor, num_classes: int,
    top_k: int, ignore_index: Optional[int], err_flag: Optional[Tensor] = None,
) -> None:
    """In-place per-class tp/fp/tn/fn with the top-k refined prediction (``mb200_multiclass_stat_scores_topk_update``)."""
    dev = require_cuda(tp, fp, tn, fn, workspace, preds, target)
    if preds.ndim != 2 or target.ndim != 1:
        raise NotImplementedError("metrics_b200: top_k > 1 supports `preds` of shape (N, C) with `target` of shape (N,)")
    preds = preds.contiguous()
    target = target.contiguous()
    with on_device(dev):
        rc = lib().mb200_multiclass_stat_scores_topk_update(
            ptr(preds), tag(preds), ptr(target), tag(target), i64(preds.shape[0]), i64(num_classes), i64(top_k),
            int(ignore_index is not None), i64(ignore_index or 0), ptr(tp), ptr(fp), ptr(tn), ptr(fn), ptr(workspace),
            ptr(err_flag), stream_handle(dev),
        )
    check(rc, "multiclass_stat_scores_topk_update")


def multiclass_stat_scores_samplewise(
    preds: Tensor, target: Tensor, num_classes: int, ignore_index: Optional[int], err_flag: Optional[Tensor] = None
):
    """Per-sample ``tp, fp, tn, fn`` of shape ``[N, C]`` over the trailing dims (``mb200_multiclass_stat_scores_samplewise``)."""
    dev = require_cuda(preds, target)
    has_class_dim = preds.ndim == target.ndim + 1
    preds = preds.contiguous()
    target = target.contiguous()
    n_outer = target.shape[0]
    inner = target.numel() // max(1, n_outer)
    counts = torch.zeros((3, n_outer, num_classes), dtype=torch.int64, device=dev)
    n_valid = torch.zeros(n_outer, dtype=torch.int64, device=dev)
    with on_device(dev):
        rc = lib().mb200_multiclass_stat_scores_samplewise(
            ptr(preds), tag(preds), int(has_class_dim), ptr(target), tag(target), i64(n_outer), i64(num_classes),
            i64(max(1, inner)), int(ignore_index is not None), i64(ignore_index or 0), ptr(counts), ptr(n_valid),
            ptr(err_flag), stream_handle(dev),
        )
    check(rc, "multiclass_stat_scores_samplewise")
    tp, fp, fn = counts[0], counts[1], counts[2]
    tn = n_valid[:, None] - tp - fp - fn
    return tp, fp, tn, fn


# ----------------------------------------------------------------------------------------------------------
# class-sharded multi-GPU curve evaluation: packing and sort+scan as separate steps
# ----------------------------------------------------------------------------------------------------------
def curve_pack_keys(preds: Tensor, rows_out: Optional[int] = None) -> Tensor:
    """Class-major sort keys of ``[n, C]`` scores: int32 ``[rows_out >= C, n]`` (rows beyond ``C`` are zero padding)."""
    dev = require_cuda(preds)
    preds = preds.contiguous()
    n, c = preds.shape
    rows = c if rows_out is None else rows_out
    keys = torch.zeros((rows, n), dtype=torch.int32, device=dev) if rows > c else torch.empty((rows, n), dtype=torch.int32, device=dev)
    with on_device(dev):
        rc = lib().mb200_curve_pack_keys(ptr(preds), tag(preds), i64(n), i64(c), ptr(keys), stream_handle(dev))
    check(rc, "curve_pack_keys")
    return keys


def curve_evaluate_keys(keys: Tensor, target: Tensor, first_class: int, nonneg: bool = False):
    """Sort + scan of packed keys ``[S, n]`` (sorted in place); positives of row ``s`` are ``target == first_class + s``.
    ``nonneg``: the keys come from non-negative (or NaN) scores — metric states — and sort as 4-byte records with the label in
    bit 0 (``mb200_curve_evaluate_keys_nonneg``)."""
    dev = require_cuda(keys, target)
    assert keys.is_contiguous() and keys.dtype == torch.int32
    target = target.contiguous()
    s, n = keys.shape
    lib_ = lib()
    nbytes = int(lib_.mb200_curve_workspace_bytes(i64(s), i64(n)))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    auroc = torch.empty(s, dtype=torch.float32, device=dev)
    ap = torch.empty(s, dtype=torch.float32, device=dev)
    counts = torch.empty((s, 3), dtype=torch.int64, device=dev)
    with on_device(dev):
        rc = (lib_.mb200_curve_evaluate_keys_nonneg if nonneg else lib_.mb200_curve_evaluate_keys)(
            ptr(keys), ptr(target), tag(target), i64(n), i64(s), i64(first_class), ptr(ws), i64(nbytes), ptr(auroc), ptr(ap),
            ptr(counts), ptr(None), stream_handle(dev),
        )
    check(rc, "curve_evaluate_keys")
    return auroc, ap, counts


def curve_evaluate_multilabel(preds: Tensor, target: Tensor, num_labels: int, ignore_index: Optional[int] = None,
                              want_curve: bool = False):
    """``num_labels`` independent binary curves from ``[N, L]`` scores / targets in one batched sort + scan
    (``mb200_curve_evaluate_multilabel``).  Same return layout as :func:`curve_evaluate`."""
    dev = require_cuda(preds, target)
    preds = preds.contiguous()
    target = target.contiguous()
    n = preds.shape[0]
    lib_ = lib()
    nbytes = int(lib_.mb200_curve_workspace_bytes_for(i64(num_labels), i64(n), tag(preds)))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    auroc = torch.empty(num_labels, dtype=torch.float32, device=dev)
    ap = torch.empty(num_labels, dtype=torch.float32, device=dev)
    counts = torch.empty((num_labels, 3), dtype=torch.int64, device=dev)
    curve = None
    if want_curve:
        thr_dtype = torch.float64 if preds.dtype == torch.float64 else torch.float32
        curve = tuple(torch.empty((num_labels, n), dtype=dt, device=dev) for dt in (torch.float32, torch.float32, thr_dtype))
    with on_device(dev):
        rc = lib_.mb200_curve_evaluate_multilabel(
            ptr(preds), tag(preds), ptr(target), tag(target), i64(n), i64(num_labels),
            ctypes.c_int(0 if ignore_index is None else 1), i64(0 if ignore_index is None else ignore_index), ptr(ws),
            i64(nbytes), ptr(auroc), ptr(ap), ptr(counts), ptr(curve[0] if curve else None),
            ptr(curve[1] if curve else None), ptr(curve[2] if curve else None), ptr(None), stream_handle(dev),
        )
    check(rc, "curve_evaluate_multilabel")
    return auroc, ap, counts, curve


# ----------------------------------------------------------------------------------------------------------
# K14 wrappers (calibration error, include/metrics_b200_calibration.h)
# ----------------------------------------------------------------------------------------------------------
def calibration_top_label(preds: Tensor, target: Tensor, ignore_index: Optional[int] = None,
                          err_flag: Optional[Tensor] = None) -> tuple[Tensor, Tensor]:
    """K14a (``mb200_calibration_top_label``): ``normalize_logits_if_needed(preds, "softmax").max(dim=1)`` and the
    ``argmax == target`` hit of every row of ``preds [N, C]`` / ``target [N]``, from one read of ``preds``.  Returns float32
    ``(confidence [N], accuracy [N])``; rows whose target is ``ignore_index`` take no part in the logits vote and hold
    zeros.  No host synchronisation."""
    dev = require_cuda(preds, target)
    preds = preds.contiguous()
    target = target.contiguous()
    n, c = preds.shape
    conf = torch.empty(n, dtype=torch.float32, device=dev)
    acc = torch.empty(n, dtype=torch.float32, device=dev)
    if n == 0:
        return conf, acc
    lib_ = lib()
    nbytes = int(lib_.mb200_calibration_scratch_bytes(n))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    with on_device(dev):
        rc = lib_.mb200_calibration_top_label(
            preds.data_ptr(), tag(preds), target.data_ptr(), tag(target), n, c, int(ignore_index is not None),
            int(ignore_index or 0), conf.data_ptr(), acc.data_ptr(), scratch.data_ptr(), nbytes, ptr(err_flag),
            stream_handle(dev),
        )
    if rc:
        check(rc, "calibration_top_label")
    return conf, acc


def calibration_bin_sums(confidences: Tensor, accuracies: Tensor, boundaries: Tensor) -> tuple[Tensor, Tensor, Tensor]:
    """K14b (``mb200_calibration_bin_sums``): per slot of ``torch.bucketize(confidences, boundaries, right=True) - 1`` the
    exact count (int64) and the float64 sums of the confidences and of the accuracies (rounded to the confidence dtype
    first).  ``boundaries`` holds ``n_bins + 1`` values in the confidence dtype; all three outputs have ``n_bins + 1`` slots.
    Deterministic: same inputs, same bits."""
    dev = require_cuda(confidences, accuracies, boundaries)
    confidences = confidences.contiguous()
    accuracies = accuracies.contiguous()
    boundaries = boundaries.contiguous()
    n, slots = confidences.numel(), boundaries.numel()
    count = torch.empty(slots, dtype=torch.int64, device=dev)
    sum_conf = torch.empty(slots, dtype=torch.float64, device=dev)
    sum_acc = torch.empty(slots, dtype=torch.float64, device=dev)
    lib_ = lib()
    nbytes = int(lib_.mb200_calibration_bin_scratch_bytes(n, slots - 1))
    scratch = torch.empty(max(nbytes, 0), dtype=torch.uint8, device=dev)
    with on_device(dev):
        rc = lib_.mb200_calibration_bin_sums(
            confidences.data_ptr(), tag(confidences), accuracies.data_ptr(), tag(accuracies), n, boundaries.data_ptr(),
            slots - 1, count.data_ptr(), sum_conf.data_ptr(), sum_acc.data_ptr(), scratch.data_ptr(), nbytes,
            stream_handle(dev),
        )
    if rc:
        check(rc, "calibration_bin_sums")
    return count, sum_conf, sum_acc


# ----------------------------------------------------------------------------------------------------------
# K15 wrapper (segmentation overlap counts, include/metrics_b200_segmentation.h)
# ----------------------------------------------------------------------------------------------------------
SEG_PREDS_NEGATIVE, SEG_PREDS_TOO_LARGE, SEG_TARGET_NEGATIVE, SEG_TARGET_TOO_LARGE = 1, 2, 4, 8
_SEG_FLOAT = (torch.float32, torch.float16, torch.bfloat16)


def _dense(strides, shape, step: int) -> bool:
    """Do these dimensions hold a row-major block whose innermost stride is ``step``?  (Size-1 dimensions never move.)"""
    for size, stride in zip(reversed(shape), reversed(strides)):
        if size != 1 and stride != step:
            return False
        step *= size
    return True


def _one_hot_layout(x: Tensor) -> Optional[tuple[int, int]]:
    """(layout, batch stride) when ``x [N, C, ...]`` can be read in place: planar (0: each sample a contiguous ``[C, S]``
    block) or channels-last (1: each sample a row-major ``[S, C]`` block, what ``one_hot(x).movedim(-1, 1)`` gives); else
    None."""
    st, shape = x.stride(), x.shape
    batch = st[0] if shape[0] > 1 else x[0].numel()
    if _dense(st[1:], shape[1:], 1):
        return 0, batch
    if (shape[1] == 1 or st[1] == 1) and _dense(st[2:], shape[2:], shape[1]):
        return 1, batch
    return None


def segmentation_overlap_counts(preds: Tensor, target: Tensor, num_classes: int, index_format: bool, mul: bool,
                                drop_background: bool, err_flag: Optional[Tensor] = None) -> Tensor:
    """K15 (``mb200_segmentation_overlap_counts``): per-sample, per-class ``(intersection, pred_sum, target_sum)`` as one
    ``[3, N, C']`` tensor, ``C' = C - 1`` when ``drop_background`` and ``C > 1``.

    Index format: ``preds``, ``target`` int64 labels ``[N, ...]``, ``C = num_classes``; out-of-range labels are left out
    and OR ``SEG_*`` bits into ``err_flag`` (int32 ``[1]``).  One-hot format: ``[N, C, ...]`` of one dtype, ``C =
    preds.shape[1]``, read in place when planar or channels-last; the intersection sums ``preds * target`` (``mul``) or
    ``preds & target`` in the input dtype.  Integer inputs give int64 counts; float inputs give float64 sums (split over
    many CTAs, folded in a fixed order: deterministic), which the caller rounds to the input dtype.  No host
    synchronisation."""
    dev = require_cuda(preds, target)
    n = preds.shape[0]
    if index_format:
        c = int(num_classes)
        preds = preds.contiguous()
        target = target.contiguous()
        inner = preds[0].numel() if n else 0
        layout, p_sn, t_sn = 0, inner, inner
    else:
        c = preds.shape[1]
        inner = preds[0, 0].numel() if n and c else 0
        pl, tl = _one_hot_layout(preds), _one_hot_layout(target)
        if pl is None or tl is None or pl[0] != tl[0]:
            preds, target = preds.contiguous(), target.contiguous()
            pl, tl = (0, c * inner), (0, c * inner)
        layout, p_sn, t_sn = pl[0], pl[1], tl[1]
    cp = c - 1 if drop_background and c > 1 else c
    out_dtype = torch.float64 if preds.dtype in _SEG_FLOAT else torch.int64
    counts = torch.empty((3, n, cp), dtype=out_dtype, device=dev)
    fmt, drop, lib_ = 0 if index_format else 1, int(bool(drop_background)), lib()
    nbytes = int(lib_.mb200_segmentation_scratch_bytes(n, c, inner, fmt, layout, tag(preds), drop))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes > 0 else None
    with on_device(dev):
        rc = lib_.mb200_segmentation_overlap_counts(
            preds.data_ptr(), tag(preds), target.data_ptr(), tag(target), n, c, inner, fmt, layout, p_sn, t_sn,
            int(bool(mul)), drop, counts.data_ptr(), ptr(scratch), max(nbytes, 0), ptr(err_flag), stream_handle(dev),
        )
    if rc:
        check(rc, "segmentation_overlap_counts")
    return counts


# ----------------------------------------------------------------------------------------------------------
# K16 wrappers (retrieval, include/metrics_b200_retrieval.h)
# ----------------------------------------------------------------------------------------------------------
RET_AP, RET_RR, RET_PRECISION, RET_RECALL, RET_HIT_RATE, RET_FALL_OUT, RET_R_PRECISION, RET_NDCG = range(8)
RET_MAX_ELEMENTS = (1 << 30) - 1


def _nbytes(v: int) -> int:
    return (int(v).bit_length() + 7) // 8


class RetrievalGroups:
    """Records sorted by (index, score descending, position) and the query boundaries: the output of one group sort."""

    def __init__(self, keys: Tensor, target: Tensor, offsets: Tensor, info: Tensor, num_queries: int, segment_bytes: int):
        self.keys, self.target, self.offsets, self.info = keys, target, offsets, info
        self.num_queries, self.segment_bytes = num_queries, segment_bytes


def retrieval_sort_scratch_bytes(n: int, index_bytes: int) -> int:
    """Workspace of the group sort; raises ValueError above 2^30 - 1 records (the radix sort counts in 30 bits)."""
    nbytes = int(lib().mb200_retrieval_sort_scratch_bytes(int(n), int(index_bytes)))
    if nbytes < 0:
        raise ValueError(f"metrics_b200: retrieval metrics support at most 2^30 - 1 = {RET_MAX_ELEMENTS} elements in total, "
                         f"got {n}.")
    return nbytes


def retrieval_sort(indexes: Optional[Tensor], preds: Tensor, target: Tensor) -> RetrievalGroups:
    """K16a + K16b: group ``preds`` / ``target`` by ``indexes`` (``None``: one query) in ascending index order, each query by
    descending score, ties in input order.  Reads the index range and the query count back (two host synchronisations;
    one when ``indexes`` is None)."""
    dev = require_cuda(preds, target) if indexes is None else require_cuda(indexes, preds, target)
    n = preds.numel()
    preds = preds.reshape(-1).to(torch.float32).contiguous()
    target = target.reshape(-1)
    target = (target.to(torch.float32) if target.is_floating_point() else target.to(torch.int64)).contiguous()
    lib_ = lib()
    retrieval_sort_scratch_bytes(n, 0)  # the size guard, before anything is allocated
    st = stream_handle(dev)
    if indexes is None:
        indexes = torch.zeros(n, dtype=torch.int64, device=dev)
        lo, hi = 0, 0
    else:
        indexes = indexes.reshape(-1).to(torch.int64).contiguous()
        rng = torch.empty(2, dtype=torch.int64, device=dev)
        with on_device(dev):
            check(lib_.mb200_retrieval_index_range(indexes.data_ptr(), n, rng.data_ptr(), st), "retrieval_index_range")
        lo, hi = rng.tolist()
    index_bytes = _nbytes(hi - lo)
    nbytes = retrieval_sort_scratch_bytes(n, index_bytes)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    keys = torch.empty(n, dtype=torch.int64, device=dev)
    sorted_target = torch.empty(n, dtype=torch.float32, device=dev)
    offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
    info = torch.zeros(2, dtype=torch.int64, device=dev)
    with on_device(dev):
        rc = lib_.mb200_retrieval_sort(indexes.data_ptr(), preds.data_ptr(), target.data_ptr(), tag(target), n, lo, hi,
                                       keys.data_ptr(), sorted_target.data_ptr(), offsets.data_ptr(), info.data_ptr(),
                                       scratch.data_ptr(), nbytes, st)
    check(rc, "retrieval_sort")
    q, flags = info.tolist()
    if flags & FLAG_SPIN_TIMEOUT:
        raise NativeLibraryError("metrics_b200.retrieval_sort: the radix sort's look-back wait expired (results invalid)")
    segment_bytes = index_bytes if index_bytes <= 4 else _nbytes(q - 1)
    return RetrievalGroups(keys, sorted_target, offsets, info, int(q), segment_bytes)


def retrieval_sort_ideal(groups: RetrievalGroups) -> Tensor:
    """K16c: every query's targets in descending order (the ideal ranking of NDCG), float32 ``[n]``."""
    dev = groups.keys.device
    n = groups.keys.numel()
    lib_ = lib()
    nbytes = int(lib_.mb200_retrieval_ideal_scratch_bytes(n, groups.segment_bytes))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    ideal = torch.empty(n, dtype=torch.float32, device=dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    with on_device(dev):
        rc = lib_.mb200_retrieval_sort_ideal(groups.keys.data_ptr(), groups.target.data_ptr(), n, groups.segment_bytes,
                                             ideal.data_ptr(), scratch.data_ptr(), nbytes, err.data_ptr(), stream_handle(dev))
    check(rc, "retrieval_sort_ideal")
    return ideal


def retrieval_evaluate(groups: RetrievalGroups, kind: int, top_k: Optional[int] = None, adaptive_k: bool = False,
                       ideal: Optional[Tensor] = None) -> tuple[Tensor, Tensor]:
    """K16d: ``(value float32 [Q], empty bool [Q])`` of metric ``kind`` per query, in ascending index order.  ``top_k``
    None (or 0) means the query length.  No host synchronisation."""
    dev = groups.keys.device
    n = groups.keys.numel()
    q = groups.num_queries
    lib_ = lib()
    nbytes = int(lib_.mb200_retrieval_evaluate_scratch_bytes(n))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    value = torch.empty(max(q, 1), dtype=torch.float32, device=dev)
    empty = torch.empty(max(q, 1), dtype=torch.uint8, device=dev)
    with on_device(dev):
        rc = lib_.mb200_retrieval_evaluate(groups.keys.data_ptr(), groups.target.data_ptr(), ptr(ideal), groups.offsets.data_ptr(),
                                           groups.info.data_ptr(), n, int(kind), int(top_k or 0), int(bool(adaptive_k)),
                                           value.data_ptr(), empty.data_ptr(), scratch.data_ptr(), nbytes, stream_handle(dev))
    check(rc, "retrieval_evaluate")
    return value[:q], empty[:q].bool()


def retrieval_auroc(groups: RetrievalGroups, top_k: Optional[int] = None, max_fpr: Optional[float] = None) -> tuple[Tensor, Tensor]:
    """K16e: ``(value float32 [Q], empty bool [Q])``: the AUROC of each query's top ``top_k`` records (None: all), the
    partial, McClish-standardised area up to ``max_fpr`` unless it is None or 1.  No host synchronisation."""
    dev = groups.keys.device
    n = groups.keys.numel()
    q = groups.num_queries
    lib_ = lib()
    nbytes = int(lib_.mb200_retrieval_evaluate_scratch_bytes(n))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    value = torch.empty(max(q, 1), dtype=torch.float32, device=dev)
    empty = torch.empty(max(q, 1), dtype=torch.uint8, device=dev)
    with on_device(dev):
        rc = lib_.mb200_retrieval_auroc(groups.keys.data_ptr(), groups.target.data_ptr(), groups.offsets.data_ptr(),
                                        groups.info.data_ptr(), n, int(top_k or 0), -1.0 if max_fpr is None else float(max_fpr),
                                        value.data_ptr(), empty.data_ptr(), scratch.data_ptr(), nbytes, stream_handle(dev))
    check(rc, "retrieval_auroc")
    return value[:q], empty[:q].bool()


def retrieval_pr_curve(groups: RetrievalGroups, max_k: int, adaptive_k: bool = False) -> tuple[Tensor, Tensor, Tensor]:
    """K16f: ``(precision float32 [Q, max_k], recall float32 [Q, max_k], empty bool [Q])`` at k = 1..max_k per query; the
    rows of queries without a positive target are zeros.  No host synchronisation."""
    dev = groups.keys.device
    n = groups.keys.numel()
    q = groups.num_queries
    lib_ = lib()
    nbytes = int(lib_.mb200_retrieval_pr_curve_scratch_bytes(n))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    precision = torch.empty((max(q, 1), max_k), dtype=torch.float32, device=dev)
    recall = torch.empty((max(q, 1), max_k), dtype=torch.float32, device=dev)
    empty = torch.empty(max(q, 1), dtype=torch.uint8, device=dev)
    with on_device(dev):
        rc = lib_.mb200_retrieval_pr_curve(groups.keys.data_ptr(), groups.target.data_ptr(), groups.offsets.data_ptr(),
                                           groups.info.data_ptr(), n, int(max_k), int(bool(adaptive_k)), precision.data_ptr(),
                                           recall.data_ptr(), empty.data_ptr(), scratch.data_ptr(), nbytes, stream_handle(dev))
    check(rc, "retrieval_pr_curve")
    return precision[:q], recall[:q], empty[:q].bool()


# ----------------------------------------------------------------------------------------------------------
# K17 wrappers (rank correlations, include/metrics_b200_rankcorr.h)
# ----------------------------------------------------------------------------------------------------------
RANKCORR_MAX_ROWS = (1 << 30) - 1
KENDALL_VARIANT = {"a": 0, "b": 1, "c": 2}
KENDALL_ALTERNATIVE = {None: 0, "two-sided": 1, "less": 2, "greater": 3}
_RANKABLE = (torch.float32, torch.float16, torch.bfloat16, torch.float64, torch.int32, torch.int64)


def rankcorr_scratch_bytes(n: int, d: int, kendall: bool) -> int:
    """Workspace of one K17 call; raises ValueError from 2^30 rows on (the radix sort counts in 30 bits)."""
    nbytes = int(lib().mb200_rankcorr_scratch_bytes(int(n), int(d), int(bool(kendall))))
    if nbytes < 0:
        raise ValueError(f"metrics_b200: rank correlations support at most 2^30 - 1 = {RANKCORR_MAX_ROWS} rows per column, "
                         f"got {n} rows x {d} columns.")
    return nbytes


def _rank_columns(x: Tensor) -> Tensor:
    """``[N]`` or ``[N, d]`` as a contiguous row-major tensor of a dtype the kernel ranks (other integer types and bool
    are widened to int64, which keeps their order)."""
    if x.dtype not in _RANKABLE:
        x = x.to(torch.int64)
    return x.contiguous()


def _rankcorr_launch(preds: Tensor, target: Tensor, kendall: bool):
    dev = require_cuda(preds, target)
    n = preds.shape[0] if preds.ndim else 1
    d = preds.shape[1] if preds.ndim == 2 else 1
    nbytes = rankcorr_scratch_bytes(n, d, kendall)  # the size guard, before anything is allocated
    preds, target = _rank_columns(preds), _rank_columns(target)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    return dev, n, d, preds, target, scratch, err


def _check_sort_flag(err: Tensor, what: str) -> None:
    if int(err.item()) & FLAG_SPIN_TIMEOUT:
        raise NativeLibraryError(f"metrics_b200.{what}: the radix sort's look-back wait expired (results invalid)")


def spearman_corrcoef(preds: Tensor, target: Tensor, out_dtype: torch.dtype, eps: float = 1e-6) -> Tensor:
    """K17: Spearman's rho of every column of ``preds`` / ``target`` (``[N]`` or ``[N, d]``, floating point), ``[d]`` in
    ``out_dtype`` (a scalar for 1-d inputs).  One host synchronisation: the sort's error flag."""
    dev, n, d, preds, target, scratch, err = _rankcorr_launch(preds, target, kendall=False)
    out = torch.empty(d, dtype=out_dtype, device=dev)
    with on_device(dev):
        rc = lib().mb200_spearman_corrcoef(preds.data_ptr(), tag(preds), target.data_ptr(), tag(target), n, d, out.data_ptr(),
                                           tag(out), float(eps), scratch.data_ptr(), scratch.numel(), err.data_ptr(), stream_handle(dev))
    check(rc, "spearman_corrcoef")
    _check_sort_flag(err, "spearman_corrcoef")
    return out.reshape(()) if preds.ndim == 1 else out


def kendall_rank_corrcoef(preds: Tensor, target: Tensor, variant: str, alternative: Optional[str]) -> tuple[Tensor, Optional[Tensor]]:
    """K17: Kendall's tau (``variant`` "a", "b" or "c") of every column and, unless ``alternative`` is None, the p-value of
    its t-test; ``[d]``, scalars when d == 1.  The p-value is float32, and so is tau except for variant "c", which has the
    promoted floating dtype of the inputs (as in the reference).  One host synchronisation: the sort's error flag."""
    tau_dtype = torch.promote_types(preds.dtype, target.dtype) if variant == "c" else torch.float32
    if not tau_dtype.is_floating_point:
        tau_dtype = torch.float32
    dev, n, d, preds, target, scratch, err = _rankcorr_launch(preds, target, kendall=True)
    tau = torch.empty(d, dtype=tau_dtype, device=dev)
    p_value = None if alternative is None else torch.empty(d, dtype=torch.float32, device=dev)
    with on_device(dev):
        rc = lib().mb200_kendall_rank_corrcoef(preds.data_ptr(), tag(preds), target.data_ptr(), tag(target), n, d,
                                               KENDALL_VARIANT[variant], KENDALL_ALTERNATIVE[alternative], tau.data_ptr(),
                                               tag(tau), ptr(p_value), scratch.data_ptr(), scratch.numel(), err.data_ptr(),
                                               stream_handle(dev))
    check(rc, "kendall_rank_corrcoef")
    _check_sort_flag(err, "kendall_rank_corrcoef")
    if d == 1:
        tau = tau.reshape(())
        p_value = None if p_value is None else p_value.reshape(())
    return tau, p_value


# ----------------------------------------------------------------------------------------------------------
# K18 wrapper (panoptic quality, include/metrics_b200_panoptic.h)
# ----------------------------------------------------------------------------------------------------------
PQ_UNKNOWN_PREDS = 1  # with FLAG_CAPACITY, the bits of K18's error word
# per-image hash-table slots of the first pass: an image with up to 1024 distinct pred or target colors and 4096 color pairs
# fits; a larger one sets FLAG_CAPACITY and the update is repeated with tables that cannot fill
PANOPTIC_COLOR_CAPACITY, PANOPTIC_PAIR_CAPACITY = 2048, 8192
PANOPTIC_RERUN_BYTES = 1 << 30  # hash tables of one launch of that repeat, at least one image
PANOPTIC_MAX_PIXELS = 1 << 30


def _pow2_at_least(v: int) -> int:
    return 1 << max(6, (int(v) - 1).bit_length())


def panoptic_categories(things, stuffs, device) -> Tensor:
    """The ``categories`` argument of K18: the category ids in ascending order, then the continuous id of each (things in
    ascending id order first, then stuffs), int64 on ``device``."""
    cid = {c: i for i, c in enumerate(sorted(things))}
    cid.update({c: len(things) + i for i, c in enumerate(sorted(stuffs))})
    ids = sorted(cid)
    return torch.tensor(ids + [cid[c] for c in ids], dtype=torch.int64, device=device)


def _pair_rows(x: Tensor) -> Tensor:
    """``[n, ..., 2]`` as a contiguous tensor whose start is aligned to one (category, instance) pair."""
    x = x.contiguous()
    if x.data_ptr() % (2 * x.element_size()):
        x = x.clone()
    return x


def panoptic_update_(iou_sum: Tensor, true_positives: Tensor, false_positives: Tensor, false_negatives: Tensor, preds: Tensor,
                     target: Tensor, categories: Tensor, num_things: int, modified: bool, allow_unknown_preds: bool) -> bool:
    """K18 (``mb200_panoptic_update``): add one batch of ``[n, *spatial, 2]`` integer panoptic maps to the four ``[K]``
    states in place.  Returns True, with the states unchanged, when ``preds`` holds a category that is neither a thing nor
    a stuff and ``allow_unknown_preds`` is False.  One host synchronisation: the error word; an image with more distinct
    segments than the first pass's tables is counted again with tables sized for one segment per pixel."""
    dev = require_cuda(preds, target, iou_sum)
    n = preds.shape[0]
    pixels = 1
    for s in preds.shape[1:-1]:
        pixels *= s
    if pixels > PANOPTIC_MAX_PIXELS:
        raise ValueError(f"metrics_b200: panoptic quality supports at most 2^30 points per image, got {pixels}.")
    preds, target = _pair_rows(preds), _pair_rows(target)
    k = categories.numel() // 2
    err = torch.empty(1, dtype=torch.int32, device=dev)
    lib_ = lib()

    def run(per_launch: int, color_capacity: int, pair_capacity: int) -> None:
        nbytes = int(lib_.mb200_panoptic_scratch_bytes(n, pixels, k, per_launch, color_capacity, pair_capacity, tag(preds),
                                                       tag(target)))
        if nbytes < 0:
            raise ValueError(f"metrics_b200: unsupported panoptic inputs ({preds.dtype}, {target.dtype}, {k} categories)")
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        with on_device(dev):
            rc = lib_.mb200_panoptic_update(preds.data_ptr(), tag(preds), target.data_ptr(), tag(target), n, pixels,
                                            categories.data_ptr(), k, int(num_things), int(bool(modified)),
                                            int(bool(allow_unknown_preds)), per_launch, color_capacity, pair_capacity,
                                            iou_sum.data_ptr(), true_positives.data_ptr(), false_positives.data_ptr(),
                                            false_negatives.data_ptr(), scratch.data_ptr(), nbytes, err.data_ptr(),
                                            stream_handle(dev))
        check(rc, "panoptic_update")

    worst = _pow2_at_least(2 * max(pixels, 1))
    run(max(n, 1), min(PANOPTIC_COLOR_CAPACITY, worst), min(PANOPTIC_PAIR_CAPACITY, worst))
    flags = int(err.item())
    if flags & PQ_UNKNOWN_PREDS:
        return True
    if flags & FLAG_CAPACITY:
        per_image = int(lib_.mb200_panoptic_scratch_bytes(1, pixels, k, 1, worst, worst, tag(preds), tag(target)))
        run(max(1, min(n, PANOPTIC_RERUN_BYTES // per_image)), worst, worst)
    return False


# ----------------------------------------------------------------------------------------------------------
# K19 wrapper (Hausdorff distance, include/metrics_b200_hausdorff.h)
# ----------------------------------------------------------------------------------------------------------
HD_PREDS_NOT_BINARY, HD_TARGET_NOT_BINARY, HD_NO_EDGES = 0, 1, 2
HD_METRICS = {"euclidean": 0, "chessboard": 1, "taxicab": 2}
# scratch of one launch: pairs are processed as many at a time as fit, at least one
HAUSDORFF_SCRATCH_BYTES = 1 << 28


def hausdorff_distance(preds: Tensor, target: Tensor, num_classes: int, index_format: bool, drop_background: bool,
                       distance_metric: str, spacing: tuple, directed: bool) -> tuple[Tensor, Tensor]:
    """K19 (``mb200_hausdorff_distance``): the ``[N, C']`` float32 Hausdorff distances of 2-D masks and the int64 ``[2]``
    error word, read in place through their strides.  Index format: int64 labels ``[N, H, W]``, ``C = num_classes``.
    One-hot format: ``[N, C, H, W]`` integer or bool tensors, ``C = preds.shape[1]``.  ``spacing``: two Python ints or
    floats; an int is int64 arithmetic, a float float32.  ``err[0]``: ``4 * pair + HD_*`` of the first failing pair, or
    -1; ``err[1]``: ``SEG_*`` label bits.  No host synchronisation."""
    dev = require_cuda(preds, target)
    n, h, w = preds.shape[0], preds.shape[-2], preds.shape[-1]
    c = int(num_classes) if index_format else preds.shape[1]
    cp = c - 1 if drop_background and c > 1 else c
    out = torch.empty((n, cp), dtype=torch.float32, device=dev)
    err = torch.empty(2, dtype=torch.int64, device=dev)
    if index_format:
        ps = (preds.stride(0), 0, preds.stride(1), preds.stride(2))
        ts = (target.stride(0), 0, target.stride(1), target.stride(2))
    else:
        ps, ts = preds.stride(), target.stride()
    int_mask = sum(1 << k for k, v in enumerate(spacing) if isinstance(v, int))
    lib_ = lib()
    per_pair = int(lib_.mb200_hausdorff_scratch_bytes(max(h, 1), max(w, 1), int(bool(directed)), 1))
    per_launch = max(1, min(n * cp, HAUSDORFF_SCRATCH_BYTES // max(per_pair, 1)))
    nbytes = int(lib_.mb200_hausdorff_scratch_bytes(max(h, 1), max(w, 1), int(bool(directed)), per_launch))
    if per_pair < 0 or nbytes < 0:
        raise ValueError(f"metrics_b200: unsupported image size {h} x {w}")
    scratch = torch.empty(nbytes if n * cp else 0, dtype=torch.uint8, device=dev)
    with on_device(dev):
        rc = lib_.mb200_hausdorff_distance(
            preds.data_ptr(), tag(preds), target.data_ptr(), tag(target), 0 if index_format else 1, n, c, h, w, *ps, *ts,
            int(bool(drop_background)), HD_METRICS[distance_metric], int_mask, float(spacing[0]), float(spacing[1]),
            int(bool(directed)), per_launch, out.data_ptr(), scratch.data_ptr(), scratch.numel(), err.data_ptr(),
            stream_handle(dev),
        )
    if rc:
        check(rc, "hausdorff_distance")
    return out, err


# ----------------------------------------------------------------------------------------------------------
# K20 wrappers (structural similarity, include/metrics_b200_image.h)
# ----------------------------------------------------------------------------------------------------------
SSIM_RANGE, SSIM_C1, SSIM_C2, SSIM_CONSTS = 0, 1, 2, 3
SSIM_MAX_TAPS = 255


def _volume(x: Tensor) -> tuple[tuple, tuple]:
    """``[b, c, d, h, w]`` and element strides of a 4-D (``d = 1``) or 5-D tensor, read in place."""
    if x.ndim == 4:
        (b, c, h, w), (sn, sc, sh, sw) = x.shape, x.stride()
        return (b, c, 1, h, w), (sn, sc, 0, sh, sw)
    return tuple(x.shape), tuple(x.stride())


def _moment_scratch(preds: Tensor, shape: tuple, taps: tuple, pads: tuple, dev) -> tuple[Tensor, int]:
    """The scratch of one windowed-moment pass (K20, K21) and its size in bytes."""
    nbytes = int(lib().mb200_ssim_scratch_bytes(tag(preds), *shape, *taps, *pads))
    if nbytes < 0:
        raise ValueError(f"metrics_b200: a filter of {tuple(taps)} taps with pads {tuple(pads)} on {tuple(shape[2:])} "
                         f"needs more than one CTA's shared memory or gives an empty output, or the batch of {shape[0]} x "
                         f"{shape[1]} planes needs 2^31 tiles or more")
    return torch.empty(nbytes, dtype=torch.uint8, device=dev), nbytes


def ssim(preds: Tensor, target: Tensor, weights: Tensor, taps: tuple, pads: tuple, crop_depth: bool,
         clamp: Optional[tuple], data_range: Optional[float], k1: float, k2: float, want_cs: bool,
         want_map: bool) -> tuple[Tensor, Optional[Tensor], Optional[Tensor]]:
    """K20: per-image float64 SSIM ``[b]``, the contrast term ``[b]`` over the crop (``want_cs``) and the map
    ``[b, c, o_d, o_h, o_w]`` in ``preds``' dtype (``want_map``).  ``taps`` / ``pads``: per axis (d, h, w); ``weights``:
    the ``sum(taps)`` filter taps in ``preds``' dtype.  ``data_range=None`` runs the data-range pre-pass first; its
    constants stay on the device.  ``target`` of any float dtype is rounded to ``preds``' dtype on load.  No host
    synchronisation."""
    dev = require_cuda(preds, target, weights)
    shape, ps = _volume(preds)
    _, ts = _volume(target)
    b = shape[0]
    lib_ = lib()
    scratch, nbytes = _moment_scratch(preds, shape, taps, pads, dev)
    sim = torch.empty(b, dtype=torch.float64, device=dev)
    cs = torch.empty(b, dtype=torch.float64, device=dev) if want_cs else None
    out_shape = (shape[0], shape[1], *(n + 2 * p - k + 1 for n, p, k in zip(shape[2:], pads, taps)))
    img = torch.empty(out_shape, dtype=preds.dtype, device=dev) if want_map else None
    stream = stream_handle(dev)
    consts = None
    with on_device(dev):
        if data_range is None:
            consts = torch.empty(SSIM_CONSTS, dtype=torch.float64, device=dev)
            rc = lib_.mb200_ssim_data_range(preds.data_ptr(), tag(preds), target.data_ptr(), tag(target), *shape, *ps, *ts,
                                            float(k1), float(k2), consts.data_ptr(), scratch.data_ptr(), nbytes, stream)
            if rc:
                check(rc, "ssim_data_range")
            c1 = c2 = 0.0
        else:
            c1, c2 = (k1 * data_range) ** 2, (k2 * data_range) ** 2
        lo, hi = clamp if clamp is not None else (0.0, 0.0)
        rc = lib_.mb200_ssim_update(
            preds.data_ptr(), tag(preds), target.data_ptr(), tag(target), *shape, *ps, *ts, *taps, *pads,
            int(bool(crop_depth)), weights.data_ptr(), int(clamp is not None), float(lo), float(hi), ptr(consts),
            float(c1), float(c2), sim.data_ptr(), ptr(cs), ptr(img), scratch.data_ptr(), nbytes, stream)
    if rc:
        check(rc, "ssim_update")
    return sim, cs, img


def ssim_avg_pool(preds: Tensor, target: Tensor, pool_depth: bool) -> tuple[Tensor, Tensor]:
    """The next MS-SSIM scale of both inputs: 2x2 (2-D) or 2x2x2 (``pool_depth``) average pool, floor sizes,
    contiguous in ``preds``' dtype (``target`` rounded to it first), shaped as the inputs' rank."""
    dev = require_cuda(preds, target)
    shape, ps = _volume(preds)
    _, ts = _volume(target)
    out = list(preds.shape[:2]) + [n // 2 for n in preds.shape[2:]]
    if not pool_depth and preds.ndim == 5:
        out[2] = preds.shape[2]
    po = torch.empty(out, dtype=preds.dtype, device=dev)
    to = torch.empty(out, dtype=preds.dtype, device=dev)
    with on_device(dev):
        rc = lib().mb200_ssim_avg_pool(preds.data_ptr(), tag(preds), target.data_ptr(), tag(target), *shape, *ps, *ts,
                                       int(bool(pool_depth)), po.data_ptr(), to.data_ptr(), stream_handle(dev))
    if rc:
        check(rc, "ssim_avg_pool")
    return po, to


# ----------------------------------------------------------------------------------------------------------
# K21 wrappers (VIF and UQI on K20's moments, include/metrics_b200_image.h)
# ----------------------------------------------------------------------------------------------------------
def vif_scale(preds: Tensor, target: Tensor, weights: Tensor, taps: tuple, eps: float,
              sigma_n_sq: float) -> tuple[Tensor, Tensor]:
    """K21, one VIF scale with valid filtering: float64 ``[b, c]`` sums of the preds term and of the target term.
    ``taps``: per axis (d, h, w); ``weights``: the ``sum(taps)`` taps in ``preds``' dtype; ``eps`` and ``sigma_n_sq``
    already rounded to that dtype.  No host synchronisation."""
    dev = require_cuda(preds, target, weights)
    shape, ps = _volume(preds)
    _, ts = _volume(target)
    scratch, nbytes = _moment_scratch(preds, shape, taps, (0, 0, 0), dev)
    sums = torch.empty(2, shape[0], shape[1], dtype=torch.float64, device=dev)
    with on_device(dev):
        rc = lib().mb200_vif_scale_update(
            preds.data_ptr(), tag(preds), target.data_ptr(), tag(target), *shape, *ps, *ts, *taps, weights.data_ptr(),
            float(eps), float(sigma_n_sq), sums[0].data_ptr(), sums[1].data_ptr(), scratch.data_ptr(), nbytes,
            stream_handle(dev))
    if rc:
        check(rc, "vif_scale_update")
    return sums[0], sums[1]


def vif_decimate(preds: Tensor, target: Tensor, weights: Tensor, taps: tuple) -> tuple[Tensor, Tensor]:
    """``conv2d(x, k)[..., ::2, ::2]`` of both 4-D inputs with the separable filter ``weights`` (``taps = (h, w)``),
    contiguous in ``preds``' dtype."""
    dev = require_cuda(preds, target, weights)
    shape, ps = _volume(preds)
    _, ts = _volume(target)
    out = (*preds.shape[:2], (preds.shape[2] - taps[0] + 2) // 2, (preds.shape[3] - taps[1] + 2) // 2)
    po = torch.empty(out, dtype=preds.dtype, device=dev)
    to = torch.empty(out, dtype=preds.dtype, device=dev)
    with on_device(dev):
        rc = lib().mb200_vif_decimate(preds.data_ptr(), tag(preds), target.data_ptr(), tag(target), *shape, *ps, *ts,
                                      *taps, weights.data_ptr(), po.data_ptr(), to.data_ptr(), stream_handle(dev))
    if rc:
        check(rc, "vif_decimate")
    return po, to


def uqi(preds: Tensor, target: Tensor, weights: Tensor, taps: tuple, pads: tuple, crop: tuple, eps: float,
        want_map: bool) -> tuple[Tensor, Optional[Tensor]]:
    """K21, UQI: per-image float64 sums ``[b]`` of the map over the crop ``[crop_h : o_h - crop_h] x
    [crop_w : o_w - crop_w]``, and the full map ``[b, c, o_d, o_h, o_w]`` in ``preds``' dtype (``want_map``).  ``taps``
    / ``pads``: per axis (d, h, w), reflect pads.  No host synchronisation."""
    dev = require_cuda(preds, target, weights)
    shape, ps = _volume(preds)
    _, ts = _volume(target)
    scratch, nbytes = _moment_scratch(preds, shape, taps, pads, dev)
    sums = torch.empty(shape[0], dtype=torch.float64, device=dev)
    out_shape = (shape[0], shape[1], *(n + 2 * p - k + 1 for n, p, k in zip(shape[2:], pads, taps)))
    img = torch.empty(out_shape, dtype=preds.dtype, device=dev) if want_map else None
    with on_device(dev):
        rc = lib().mb200_uqi_update(
            preds.data_ptr(), tag(preds), target.data_ptr(), tag(target), *shape, *ps, *ts, *taps, *pads, *crop,
            weights.data_ptr(), float(eps), sums.data_ptr(), ptr(img), scratch.data_ptr(), nbytes, stream_handle(dev))
    if rc:
        check(rc, "uqi_update")
    return sums, img
