"""ROC functionals, exact mode (reference: functional/classification/roc.py)."""
from __future__ import annotations

from typing import List, Optional, Union

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200.functional.classification.precision_recall_curve import (
    _binary_clf_curve,
    _binary_precision_recall_curve_arg_validation,
    _binary_precision_recall_curve_format,
    _binary_precision_recall_curve_tensor_validation,
    _binary_precision_recall_curve_update,
    _multiclass_precision_recall_curve_arg_validation,
    _multiclass_precision_recall_curve_format,
    _multiclass_precision_recall_curve_tensor_validation,
    _multiclass_precision_recall_curve_update,
    _ovr_curves,
    _safe_div,
)
from metrics_b200.utilities.compute import interp
from metrics_b200.utilities.prints import rank_zero_warn


def _roc_from_counts(fps: Tensor, tps: Tensor, thres: Tensor) -> tuple[Tensor, Tensor, Tensor]:
    """fpr / tpr with the (0, 0) point at threshold 1 prepended; degenerate curves give zeros + a warning
    (reference :53-78)."""
    zero = torch.zeros(1, dtype=tps.dtype, device=tps.device)
    tps = torch.cat([zero, tps])
    fps = torch.cat([zero, fps])
    thres = torch.cat([torch.ones(1, dtype=thres.dtype, device=thres.device), thres])
    if fps[-1] <= 0:
        rank_zero_warn(
            "No negative samples in targets, false positive value should be meaningless."
            " Returning zero tensor in false positive score",
            UserWarning,
        )
        fpr = torch.zeros_like(thres)
    else:
        fpr = fps / fps[-1]
    if tps[-1] <= 0:
        rank_zero_warn(
            "No positive samples in targets, true positive value should be meaningless."
            " Returning zero tensor in true positive score",
            UserWarning,
        )
        tpr = torch.zeros_like(thres)
    else:
        tpr = tps / tps[-1]
    return fpr, tpr, thres


def _binary_roc_compute(
    state: Union[Tensor, tuple[Tensor, Tensor]], thresholds: Optional[Tensor], pos_label: int = 1
) -> tuple[Tensor, Tensor, Tensor]:
    if isinstance(state, Tensor) and thresholds is not None:  # binned (reference :45-52)
        tps, fps, fns, tns = state[:, 1, 1], state[:, 0, 1], state[:, 1, 0], state[:, 0, 0]
        return _safe_div(fps, fps + tns).flip(0), _safe_div(tps, tps + fns).flip(0), thresholds.flip(0)
    fps, tps, thres = _binary_clf_curve(preds=state[0], target=state[1], pos_label=pos_label)
    return _roc_from_counts(fps, tps, thres)


def binary_roc(
    preds: Tensor,
    target: Tensor,
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
    validate_args: bool = True,
) -> tuple[Tensor, Tensor, Tensor]:
    """fpr, tpr, thresholds (descending, leading threshold 1.0) — reference :83-168."""
    if validate_args:
        _binary_precision_recall_curve_arg_validation(thresholds, ignore_index)
        _binary_precision_recall_curve_tensor_validation(preds, target, ignore_index)
    preds, target, thresholds = _binary_precision_recall_curve_format(preds, target, thresholds, ignore_index)
    state = _binary_precision_recall_curve_update(preds, target, thresholds)
    return _binary_roc_compute(state, thresholds)


def _multiclass_roc_compute(
    state: Union[Tensor, tuple[Tensor, Tensor]],
    num_classes: int,
    thresholds: Optional[Tensor],
    average: Optional[str] = None,
):
    """Per-class ROC curves from ONE batched sort (reference loops over classes, :176-181)."""
    if average == "micro":
        return _binary_roc_compute(state, thresholds, pos_label=1)
    if isinstance(state, Tensor) and thresholds is not None:  # binned (reference :171-179)
        tps, fps, fns, tns = state[:, :, 1, 1], state[:, :, 0, 1], state[:, :, 1, 0], state[:, :, 0, 0]
        tpr = _safe_div(tps, tps + fns).flip(0).T
        fpr = _safe_div(fps, fps + tns).flip(0).T
        thres = thresholds.flip(0)
        if average == "macro":
            thres = thres.repeat(num_classes).sort(descending=True).values
            mean_fpr = fpr.flatten().sort().values
            mean_tpr = torch.zeros_like(mean_fpr)
            for c in range(num_classes):
                mean_tpr += interp(mean_fpr, fpr[c], tpr[c])
            mean_tpr /= num_classes
            return mean_fpr, mean_tpr, thres
        return fpr, tpr, thres
    fps, tps, thr, lengths = _ovr_curves(state[0], state[1], num_classes)
    fpr_list, tpr_list, thres_list = [], [], []
    for c in range(num_classes):
        u = lengths[c]
        f, t, th = _roc_from_counts(fps[c, :u], tps[c, :u], thr[c, :u])
        fpr_list.append(f)
        tpr_list.append(t)
        thres_list.append(th)
    if average == "macro":
        thres = torch.cat(thres_list, dim=0).sort(descending=True).values
        mean_fpr = torch.cat(fpr_list, dim=0).sort().values
        mean_tpr = torch.zeros_like(mean_fpr)
        for c in range(num_classes):
            mean_tpr += interp(mean_fpr, fpr_list[c], tpr_list[c])
        mean_tpr /= num_classes
        return mean_fpr, mean_tpr, thres
    return fpr_list, tpr_list, thres_list


def multiclass_roc(
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    average: Optional[Literal["micro", "macro"]] = None,
    ignore_index: Optional[int] = None,
    validate_args: bool = True,
):
    """One-vs-rest ROC curves — reference :207-320."""
    if validate_args:
        _multiclass_precision_recall_curve_arg_validation(num_classes, thresholds, ignore_index, average)
        _multiclass_precision_recall_curve_tensor_validation(preds, target, num_classes, ignore_index)
    preds, target, thresholds = _multiclass_precision_recall_curve_format(
        preds, target, num_classes, thresholds, ignore_index, average
    )
    state = _multiclass_precision_recall_curve_update(preds, target, num_classes, thresholds, average)
    return _multiclass_roc_compute(state, num_classes, thresholds, average)


# ----------------------------------------------------------------------------------------------------------------------
# multilabel (reference roc.py:323-458)
# ----------------------------------------------------------------------------------------------------------------------
def _multilabel_roc_compute(
    state: Union[Tensor, tuple[Tensor, Tensor]],
    num_labels: int,
    thresholds: Optional[Tensor],
    ignore_index: Optional[int] = None,
):
    """Per-label ROC curves from ONE batched sort (reference loops over labels, :344-355)."""
    from metrics_b200.functional.classification.precision_recall_curve import _multilabel_curves

    if isinstance(state, Tensor) and thresholds is not None:
        tps, fps, fns, tns = state[:, :, 1, 1], state[:, :, 0, 1], state[:, :, 1, 0], state[:, :, 0, 0]
        return _safe_div(fps, fps + tns).flip(0).T, _safe_div(tps, tps + fns).flip(0).T, thresholds.flip(0)
    fps, tps, thr, host = _multilabel_curves(state[0], state[1], num_labels, ignore_index)
    fpr_list, tpr_list, thres_list = [], [], []
    for l in range(num_labels):
        u = host[l][2]
        f, t, th = _roc_from_counts(fps[l, :u], tps[l, :u], thr[l, :u])
        fpr_list.append(f)
        tpr_list.append(t)
        thres_list.append(th)
    return fpr_list, tpr_list, thres_list


def multilabel_roc(
    preds: Tensor,
    target: Tensor,
    num_labels: int,
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
    validate_args: bool = True,
):
    """Per-label ROC curves — reference :359-458."""
    from metrics_b200.functional.classification.precision_recall_curve import (
        _multilabel_precision_recall_curve_arg_validation,
        _multilabel_precision_recall_curve_format,
        _multilabel_precision_recall_curve_tensor_validation,
        _multilabel_precision_recall_curve_update,
    )

    if validate_args:
        _multilabel_precision_recall_curve_arg_validation(num_labels, thresholds, ignore_index)
        _multilabel_precision_recall_curve_tensor_validation(preds, target, num_labels, ignore_index)
    preds, target, thresholds = _multilabel_precision_recall_curve_format(preds, target, num_labels, thresholds, ignore_index)
    state = _multilabel_precision_recall_curve_update(preds, target, num_labels, thresholds, ignore_index)
    return _multilabel_roc_compute(state, num_labels, thresholds, ignore_index)


def roc(preds: Tensor, target: Tensor, task: Literal["binary", "multiclass", "multilabel"],
        thresholds: Optional[Union[int, List[float], Tensor]] = None, num_classes: Optional[int] = None,
        num_labels: Optional[int] = None, average: Optional[Literal["micro", "macro"]] = None,
        ignore_index: Optional[int] = None, validate_args: bool = True):
    """Task wrapper (reference :461-565)."""
    from metrics_b200.functional.classification._task import call_for_task

    return call_for_task(
        task, num_classes, num_labels,
        lambda: binary_roc(preds, target, thresholds, ignore_index, validate_args),
        lambda c: multiclass_roc(preds, target, c, thresholds, average, ignore_index, validate_args),
        lambda n: multilabel_roc(preds, target, n, thresholds, ignore_index, validate_args))
