"""Precision-recall-curve functionals, exact mode (reference: functional/classification/precision_recall_curve.py).

`_binary_clf_curve` — the sort + cumulative TP/FP scan that every curve metric is built on — is one batched GPU
pipeline here (`mb200_curve_evaluate`, csrc/curve.cu): key packing, 4-pass 8-bit LSD radix sort of (score key, label
byte), tie-collapsing integer scan.  The multiclass one-vs-rest loop of the reference (one full sort per class in
Python, :565-569) is a single call with one contiguous segment per class.

Binned mode (``thresholds`` given): the `[T, (C,) 2, 2]` multi-threshold confusion matrix of a batch comes from ONE
pass (`mb200_binned_curve_update`, csrc/binned.cu: bucket search + histogram + suffix sums) instead of the reference's
N*T(*C) temporaries or T passes (:191-251, :464-533).
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Union

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200 import _native
from metrics_b200.utilities.checks import _check_same_shape
from metrics_b200.utilities.compute import interp
from metrics_b200.utilities.prints import rank_zero_warn


def _no_binned(thresholds: Optional[Union[int, List[float], Tensor]]) -> None:
    """Kept for callers that only make sense in exact mode."""
    if thresholds is not None:
        raise ValueError("this code path expects exact mode (`thresholds=None`)")


def _safe_div(num: Tensor, denom: Tensor) -> Tensor:
    from metrics_b200.utilities.compute import _safe_divide

    return _safe_divide(num, denom)


def _binary_clf_curve(
    preds: Tensor,
    target: Tensor,
    sample_weights: Optional[Union[Sequence, Tensor]] = None,
    pos_label: int = 1,
) -> tuple[Tensor, Tensor, Tensor]:
    """``fps, tps, thresholds`` at every distinct score, descending (reference :30-82).  All three are float32 with
    integer-valued counts, exactly like the reference's ``cumsum(target * 1.0)``."""
    if preds.ndim > target.ndim:
        preds = preds[:, 0]
    if preds.numel() == 0:
        raise IndexError("metrics_b200: cannot compute a curve from zero samples")
    if sample_weights is not None:  # reference :45-46, :64, :73-78
        if not isinstance(sample_weights, Tensor):
            sample_weights = torch.tensor(sample_weights, device=preds.device, dtype=torch.float)
        fps, tps, thr = _native.curve_weighted_clf_curve(preds, target, sample_weights.to(preds.device), pos_label)
        out_dtype = torch.result_type(torch.zeros((), dtype=torch.long), sample_weights)  # `target * weight`
        if preds.dtype not in (torch.float32, torch.float64):
            thr = thr.to(preds.dtype)
        return fps.to(out_dtype), tps.to(out_dtype), thr
    _, _, counts, (fps, tps, thr) = _native.curve_evaluate(preds, target, 1, pos_label, want_curve=True)
    n_thr = int(counts[0, 2])  # data-dependent output size -> one host sync (the reference syncs in `torch.where`)
    thr = thr[0, :n_thr]
    if preds.dtype != torch.float32:
        thr = thr.to(preds.dtype)
    return fps[0, :n_thr], tps[0, :n_thr], thr


def _adjust_threshold_arg(
    thresholds: Optional[Union[int, List[float], Tensor]] = None, device: Optional[torch.device] = None
) -> Optional[Tensor]:
    if isinstance(thresholds, int):
        return torch.linspace(0, 1, thresholds, device=device)
    if isinstance(thresholds, list):
        return torch.tensor(thresholds, device=device)
    return thresholds


# ---------------------------------------------------------------------------------------------------------
# binary
# ---------------------------------------------------------------------------------------------------------
def _binary_precision_recall_curve_arg_validation(
    thresholds: Optional[Union[int, List[float], Tensor]] = None, ignore_index: Optional[int] = None
) -> None:
    if thresholds is not None and not isinstance(thresholds, (list, int, Tensor)):
        raise ValueError(
            "Expected argument `thresholds` to either be an integer, list of floats or"
            f" tensor of floats, but got {thresholds}"
        )
    if isinstance(thresholds, int) and thresholds < 2:
        raise ValueError(
            f"If argument `thresholds` is an integer, expected it to be larger than 1, but got {thresholds}"
        )
    if isinstance(thresholds, list) and not all(isinstance(t, float) and 0 <= t <= 1 for t in thresholds):
        raise ValueError(
            "If argument `thresholds` is a list, expected all elements to be floats in the [0,1] range,"
            f" but got {thresholds}"
        )
    if isinstance(thresholds, Tensor) and not thresholds.ndim == 1:
        raise ValueError("If argument `thresholds` is an tensor, expected the tensor to be 1d")
    if ignore_index is not None and not isinstance(ignore_index, int):
        raise ValueError(f"Expected argument `ignore_index` to either be `None` or an integer, but got {ignore_index}")


def _binary_precision_recall_curve_tensor_validation(
    preds: Tensor, target: Tensor, ignore_index: Optional[int] = None
) -> None:
    """Same shape, float scores, integer targets in {0, 1} (+ ignore_index) — reference :127-161."""
    _check_same_shape(preds, target)
    if target.is_floating_point():
        raise ValueError(
            "Expected argument `target` to be an int or long tensor with ground truth labels"
            f" but got tensor with dtype {target.dtype}"
        )
    if not preds.is_floating_point():
        raise ValueError(
            "Expected argument `preds` to be an floating tensor with probability/logit scores,"
            f" but got tensor with dtype {preds.dtype}"
        )
    bad = (target != 0) & (target != 1)
    if ignore_index is not None:
        bad &= target != ignore_index
    if bool(bad.any()):
        found = torch.unique(target)
        raise RuntimeError(
            f"Detected the following values in `target`: {found} but expected only"
            f" the following values {[0, 1] if ignore_index is None else [ignore_index]}."
        )


def _binary_precision_recall_curve_format(
    preds: Tensor,
    target: Tensor,
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
) -> tuple[Tensor, Tensor, Optional[Tensor]]:
    """Flatten, drop ignored samples, sigmoid if the batch holds logits (kernel K6) — reference :164-188."""
    preds = preds.flatten()
    target = target.flatten()
    if ignore_index is not None:
        keep = target != ignore_index
        preds, target = preds[keep], target[keep]
    preds = _native.sigmoid_if_logits(preds)
    return preds, target, _adjust_threshold_arg(thresholds, preds.device)


def _binary_precision_recall_curve_update(
    preds: Tensor, target: Tensor, thresholds: Optional[Tensor]
) -> Union[Tensor, tuple[Tensor, Tensor]]:
    """Exact mode: the formatted batch itself.  Binned mode: its ``[T, 2, 2]`` multi-threshold confusion matrix."""
    if thresholds is None:
        return preds, target
    return _native.binned_curve_update(preds, target, thresholds.to(preds.device), 1)


def _pr_from_counts(fps: Tensor, tps: Tensor, thr: Tensor, all_negative: bool) -> tuple[Tensor, Tensor, Tensor]:
    """precision / recall arrays of the reference from descending-threshold counts (reference :275-290)."""
    precision = tps / (tps + fps)
    recall = tps / tps[-1]
    if all_negative:
        rank_zero_warn(
            "No positive samples found in target, recall is undefined. Setting recall to one for all thresholds.",
            UserWarning,
        )
        recall = torch.ones_like(recall)
    precision = torch.cat([precision.flip(0), torch.ones(1, dtype=precision.dtype, device=precision.device)])
    recall = torch.cat([recall.flip(0), torch.zeros(1, dtype=recall.dtype, device=recall.device)])
    return precision, recall, thr.flip(0).detach().clone()


def _binary_precision_recall_curve_compute(
    state: Union[Tensor, tuple[Tensor, Tensor]], thresholds: Optional[Tensor], pos_label: int = 1
) -> tuple[Tensor, Tensor, Tensor]:
    if isinstance(state, Tensor) and thresholds is not None:  # binned (reference :265-273)
        tps, fps, fns = state[:, 1, 1], state[:, 0, 1], state[:, 1, 0]
        precision = _safe_div(tps, tps + fps)
        recall = _safe_div(tps, tps + fns)
        precision = torch.cat([precision, torch.ones(1, dtype=precision.dtype, device=precision.device)])
        recall = torch.cat([recall, torch.zeros(1, dtype=recall.dtype, device=recall.device)])
        return precision, recall, thresholds
    fps, tps, thr = _binary_clf_curve(state[0], state[1], pos_label=pos_label)
    # the reference tests `(target == 0).all()` on the raw target, whatever pos_label is (:278)
    return _pr_from_counts(fps, tps, thr, bool((state[1] == 0).all()))


def binary_precision_recall_curve(
    preds: Tensor,
    target: Tensor,
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
    validate_args: bool = True,
) -> tuple[Tensor, Tensor, Tensor]:
    """precision, recall, thresholds (ascending) for binary scores — reference :293-380."""
    if validate_args:
        _binary_precision_recall_curve_arg_validation(thresholds, ignore_index)
        _binary_precision_recall_curve_tensor_validation(preds, target, ignore_index)
    preds, target, thresholds = _binary_precision_recall_curve_format(preds, target, thresholds, ignore_index)
    state = _binary_precision_recall_curve_update(preds, target, thresholds)
    return _binary_precision_recall_curve_compute(state, thresholds)


# ---------------------------------------------------------------------------------------------------------
# multiclass
# ---------------------------------------------------------------------------------------------------------
def _multiclass_precision_recall_curve_arg_validation(
    num_classes: int,
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
    average: Optional[str] = None,
) -> None:
    if not isinstance(num_classes, int) or num_classes < 2:
        raise ValueError(f"Expected argument `num_classes` to be an integer larger than 1, but got {num_classes}")
    if average not in (None, "micro", "macro"):
        raise ValueError(f"Expected argument `average` to be one of None, 'micro' or 'macro', but got {average}")
    _binary_precision_recall_curve_arg_validation(thresholds, ignore_index)


def _multiclass_precision_recall_curve_tensor_validation(
    preds: Tensor, target: Tensor, num_classes: int, ignore_index: Optional[int] = None
) -> None:
    if not preds.ndim == target.ndim + 1:
        raise ValueError(
            f"Expected `preds` to have one more dimension than `target` but got {preds.ndim} and {target.ndim}"
        )
    if target.is_floating_point():
        raise ValueError(
            f"Expected argument `target` to be an int or long tensor, but got tensor with dtype {target.dtype}"
        )
    if not preds.is_floating_point():
        raise ValueError(f"Expected `preds` to be a float tensor, but got {preds.dtype}")
    if preds.shape[1] != num_classes:
        raise ValueError(
            "Expected `preds.shape[1]` to be equal to the number of classes but"
            f" got {preds.shape[1]} and {num_classes}."
        )
    if preds.shape[0] != target.shape[0] or preds.shape[2:] != target.shape[1:]:
        raise ValueError(
            "Expected the shape of `preds` should be (N, C, ...) and the shape of `target` should be (N, ...)"
            f" but got {preds.shape} and {target.shape}"
        )
    bad = (target < 0) | (target >= num_classes)
    if ignore_index is not None:
        bad &= target != ignore_index
    if bool(bad.any()):
        expected = num_classes if ignore_index is None else num_classes + 1
        raise RuntimeError(
            "Detected more unique values in `target` than `num_classes`. Expected only "
            f"{expected} but found values outside of [0, {num_classes}) in `target`."
        )


def _multiclass_precision_recall_curve_format(
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
    average: Optional[str] = None,
) -> tuple[Tensor, Tensor, Optional[Tensor]]:
    """``[N, C, ...] -> [N', C]``, drop ignored samples, softmax if the batch holds logits — reference :430-461."""
    preds = preds.transpose(0, 1).reshape(num_classes, -1).T
    target = target.flatten()
    if ignore_index is not None:
        keep = target != ignore_index
        preds, target = preds[keep], target[keep]
    preds = _native.softmax_if_logits(preds)
    if average == "micro":
        preds = preds.flatten()
        target = torch.nn.functional.one_hot(target, num_classes=num_classes).flatten()
    return preds, target, _adjust_threshold_arg(thresholds, preds.device)


def _multiclass_precision_recall_curve_update(
    preds: Tensor, target: Tensor, num_classes: int, thresholds: Optional[Tensor], average: Optional[str] = None
) -> Union[Tensor, tuple[Tensor, Tensor]]:
    if thresholds is None:
        return preds, target
    if average == "micro":
        return _binary_precision_recall_curve_update(preds, target, thresholds)
    return _native.binned_curve_update(preds, target, thresholds.to(preds.device), num_classes)


def _ovr_curves(preds: Tensor, target: Tensor, num_classes: int):
    """All ``num_classes`` one-vs-rest ``(fps, tps, thr)`` curves from one batched sort; per-class valid lengths."""
    _, _, counts, (fps, tps, thr) = _native.curve_evaluate(preds, target, num_classes, want_curve=True)
    lengths = counts[:, 2].tolist()  # one host sync for all classes
    if preds.dtype != torch.float32:
        thr = thr.to(preds.dtype)
    return fps, tps, thr, lengths


def _multiclass_precision_recall_curve_compute(
    state: Union[Tensor, tuple[Tensor, Tensor]],
    num_classes: int,
    thresholds: Optional[Tensor],
    average: Optional[str] = None,
):
    """Per-class PR curves (lists in exact mode, ``[C, T+1]`` tensors in binned mode) or their macro/micro aggregation
    — reference :536-589."""
    if average == "micro":
        return _binary_precision_recall_curve_compute(state, thresholds)
    if isinstance(state, Tensor) and thresholds is not None:
        tps, fps, fns = state[:, :, 1, 1], state[:, :, 0, 1], state[:, :, 1, 0]
        precision = _safe_div(tps, tps + fps)
        recall = _safe_div(tps, tps + fns)
        precision = torch.cat([precision, torch.ones(1, num_classes, dtype=precision.dtype, device=precision.device)]).T
        recall = torch.cat([recall, torch.zeros(1, num_classes, dtype=recall.dtype, device=recall.device)]).T
        if average == "macro":
            thres = thresholds.repeat(num_classes).sort().values
            mean_precision = precision.flatten().sort().values
            mean_recall = torch.zeros_like(mean_precision)
            for c in range(num_classes):
                mean_recall += interp(mean_precision, precision[c], recall[c])
            mean_recall /= num_classes
            return mean_precision, mean_recall, thres
        return precision, recall, thresholds
    fps, tps, thr, lengths = _ovr_curves(state[0], state[1], num_classes)
    all_zero = bool((state[1] == 0).all())
    precision_list, recall_list, thres_list = [], [], []
    for c in range(num_classes):
        u = lengths[c]
        p, r, t = _pr_from_counts(fps[c, :u], tps[c, :u], thr[c, :u], all_zero)
        precision_list.append(p)
        recall_list.append(r)
        thres_list.append(t)
    if average == "macro":
        thres = torch.cat(thres_list, 0).sort().values
        mean_precision = torch.cat(precision_list, 0).sort().values
        mean_recall = torch.zeros_like(mean_precision)
        for c in range(num_classes):
            mean_recall += interp(mean_precision, precision_list[c], recall_list[c])
        mean_recall /= num_classes
        return mean_precision, mean_recall, thres
    return precision_list, recall_list, thres_list


def multiclass_precision_recall_curve(
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    average: Optional[Literal["micro", "macro"]] = None,
    ignore_index: Optional[int] = None,
    validate_args: bool = True,
):
    """One-vs-rest PR curves — reference :592-700."""
    if validate_args:
        _multiclass_precision_recall_curve_arg_validation(num_classes, thresholds, ignore_index, average)
        _multiclass_precision_recall_curve_tensor_validation(preds, target, num_classes, ignore_index)
    preds, target, thresholds = _multiclass_precision_recall_curve_format(
        preds, target, num_classes, thresholds, ignore_index, average
    )
    state = _multiclass_precision_recall_curve_update(preds, target, num_classes, thresholds, average)
    return _multiclass_precision_recall_curve_compute(state, num_classes, thresholds, average)


# ----------------------------------------------------------------------------------------------------------------------
# multilabel (reference :711-941): one binary curve per label, all labels in ONE batched sort + scan
# ----------------------------------------------------------------------------------------------------------------------
def _multilabel_precision_recall_curve_arg_validation(
    num_labels: int,
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
) -> None:
    _multiclass_precision_recall_curve_arg_validation(num_labels, thresholds, ignore_index)


def _multilabel_precision_recall_curve_tensor_validation(
    preds: Tensor, target: Tensor, num_labels: int, ignore_index: Optional[int] = None
) -> None:
    _binary_precision_recall_curve_tensor_validation(preds, target, ignore_index)
    if preds.shape[1] != num_labels:
        raise ValueError(
            "Expected both `target.shape[1]` and `preds.shape[1]` to be equal to the number of labels"
            f" but got {preds.shape[1]} and expected {num_labels}"
        )


def _multilabel_precision_recall_curve_format(
    preds: Tensor,
    target: Tensor,
    num_labels: int,
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
) -> tuple[Tensor, Tensor, Optional[Tensor]]:
    """``[N, L, ...] -> [N', L]``, sigmoid if the batch holds logits — reference :745-774.  Ignored entries stay in the
    state (they are dropped per label by the kernels: exact mode gives them the largest sort key, the binned kernel skips
    targets equal to ``ignore_index`` in the target's dtype and every target that is neither 0 nor 1), so no masked copy of
    the batch is made."""
    preds = preds.transpose(0, 1).reshape(num_labels, -1).T
    target = target.transpose(0, 1).reshape(num_labels, -1).T
    preds = _native.sigmoid_if_logits(preds.contiguous())
    return preds, target.contiguous(), _adjust_threshold_arg(thresholds, preds.device)


def _multilabel_precision_recall_curve_update(
    preds: Tensor, target: Tensor, num_labels: int, thresholds: Optional[Tensor], ignore_index: Optional[int] = None
) -> Union[Tensor, tuple[Tensor, Tensor]]:
    """Exact mode keeps the batch; binned mode returns the ``[T, L, 2, 2]`` multi-threshold confusion matrix
    (reference :777-799) from the K4 kernel, which drops the entries the reference's format masks (``target ==
    ignore_index``, :766-772) — also when ``ignore_index`` is 0 or 1."""
    if thresholds is None:
        return preds, target
    # the kernel skips every target that is neither 0 nor 1 by itself: it is handed `ignore_index` only when that names label
    # 0 or 1 in the target's dtype
    extra = {"ignore_index": ignore_index} if _ignores_a_binary_label(ignore_index, target.dtype) else {}
    return _native.binned_curve_update(preds, target, thresholds.to(preds.device), num_labels, multilabel=True, **extra)


_LABEL_WIDTH = {torch.uint8: (8, False), torch.int8: (8, True), torch.int16: (16, True), torch.int32: (32, True)}


def _ignores_a_binary_label(ignore_index: Optional[int], dtype: torch.dtype) -> bool:
    """Does ``target == ignore_index`` select targets holding 0 or 1?  ATen casts the Python int to the target's dtype
    first (two's complement wrap: with uint8 targets 257 is 1); int64 and bool targets compare the value itself."""
    if ignore_index is None:
        return False
    v = int(ignore_index)
    if dtype in _LABEL_WIDTH:
        width, signed = _LABEL_WIDTH[dtype]
        v &= (1 << width) - 1
        if signed and v >= 1 << (width - 1):
            v -= 1 << width
    return v in (0, 1)


def _multilabel_curves(preds: Tensor, target: Tensor, num_labels: int, ignore_index: Optional[int]):
    _, _, counts, (fps, tps, thr) = _native.curve_evaluate_multilabel(preds, target, num_labels, ignore_index, want_curve=True)
    host = counts.tolist()  # one host sync for all labels
    if preds.dtype != torch.float32:
        thr = thr.to(preds.dtype)
    return fps, tps, thr, host


def _multilabel_precision_recall_curve_compute(
    state: Union[Tensor, tuple[Tensor, Tensor]],
    num_labels: int,
    thresholds: Optional[Tensor],
    ignore_index: Optional[int] = None,
):
    """Reference :802-836 (a Python loop over labels with a sort each)."""
    if isinstance(state, Tensor) and thresholds is not None:
        tps, fps, fns = state[:, :, 1, 1], state[:, :, 0, 1], state[:, :, 1, 0]
        precision = _safe_div(tps, tps + fps)
        recall = _safe_div(tps, tps + fns)
        precision = torch.cat([precision, torch.ones(1, num_labels, dtype=precision.dtype, device=precision.device)])
        recall = torch.cat([recall, torch.zeros(1, num_labels, dtype=recall.dtype, device=recall.device)])
        return precision.T, recall.T, thresholds
    fps, tps, thr, host = _multilabel_curves(state[0], state[1], num_labels, ignore_index)
    precision_list, recall_list, thres_list = [], [], []
    for l in range(num_labels):
        n_pos, _, u = host[l]
        p, r, t = _pr_from_counts(fps[l, :u], tps[l, :u], thr[l, :u], n_pos == 0)
        precision_list.append(p)
        recall_list.append(r)
        thres_list.append(t)
    return precision_list, recall_list, thres_list


def multilabel_precision_recall_curve(
    preds: Tensor,
    target: Tensor,
    num_labels: int,
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
    validate_args: bool = True,
):
    """Per-label PR curves — reference :839-941."""
    if validate_args:
        _multilabel_precision_recall_curve_arg_validation(num_labels, thresholds, ignore_index)
        _multilabel_precision_recall_curve_tensor_validation(preds, target, num_labels, ignore_index)
    preds, target, thresholds = _multilabel_precision_recall_curve_format(preds, target, num_labels, thresholds, ignore_index)
    state = _multilabel_precision_recall_curve_update(preds, target, num_labels, thresholds, ignore_index)
    return _multilabel_precision_recall_curve_compute(state, num_labels, thresholds, ignore_index)


def precision_recall_curve(preds: Tensor, target: Tensor, task: Literal["binary", "multiclass", "multilabel"],
                           thresholds: Optional[Union[int, List[float], Tensor]] = None, num_classes: Optional[int] = None,
                           num_labels: Optional[int] = None, average: Optional[Literal["micro", "macro"]] = None,
                           ignore_index: Optional[int] = None, validate_args: bool = True):
    """Task wrapper (reference :944-1014)."""
    from metrics_b200.functional.classification._task import call_for_task

    return call_for_task(
        task, num_classes, num_labels,
        lambda: binary_precision_recall_curve(preds, target, thresholds, ignore_index, validate_args),
        lambda c: multiclass_precision_recall_curve(preds, target, c, thresholds, average, ignore_index, validate_args),
        lambda n: multilabel_precision_recall_curve(preds, target, n, thresholds, ignore_index, validate_args))
