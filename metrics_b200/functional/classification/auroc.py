"""AUROC functionals, exact mode (reference: functional/classification/auroc.py).

``max_fpr=None``: the area comes straight out of the scan kernel as the exact integer ``sum dFP * (TP_prev + TP)``
divided by ``2 * P * N`` in fp64 (the reference builds fpr/tpr in fp32 and calls trapz).  ``max_fpr`` given: the curve
is materialised and the reference's partial-AUC + McClish correction is applied to it.
"""
from __future__ import annotations

from typing import List, Optional, Union

import torch
from torch import Tensor, tensor
from typing_extensions import Literal

from metrics_b200 import _native
from metrics_b200.functional.classification.precision_recall_curve import (
    _binary_precision_recall_curve_arg_validation,
    _binary_precision_recall_curve_format,
    _binary_precision_recall_curve_tensor_validation,
    _binary_precision_recall_curve_update,
    _multiclass_precision_recall_curve_arg_validation,
    _multiclass_precision_recall_curve_format,
    _multiclass_precision_recall_curve_tensor_validation,
    _multiclass_precision_recall_curve_update,
)
from metrics_b200.functional.classification.roc import _binary_roc_compute, _multiclass_roc_compute
from metrics_b200.utilities.compute import _auc_compute_without_check, _safe_divide
from metrics_b200.utilities.prints import rank_zero_warn


def _reduce_per_class(res: Tensor, average: Optional[str], weights: Optional[Tensor], what: str) -> Tensor:
    """none / macro / weighted reduction over classes, ignoring NaN classes (reference auroc.py:45-70)."""
    if average is None or average == "none":
        return res
    nan = torch.isnan(res)
    if bool(nan.any()):
        rank_zero_warn(
            f"{what} score for one or more classes was `nan`. Ignoring these classes in {average}-average",
            UserWarning,
        )
    keep = ~nan
    if average == "macro":
        return res[keep].mean()
    if average == "weighted" and weights is not None:
        w = _safe_divide(weights[keep], weights[keep].sum())
        return (res[keep] * w).sum()
    raise ValueError("Received an incompatible combinations of inputs to make reduction.")


def _binary_auroc_arg_validation(
    max_fpr: Optional[float] = None,
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
) -> None:
    _binary_precision_recall_curve_arg_validation(thresholds, ignore_index)
    if max_fpr is not None and not isinstance(max_fpr, float) and 0 < max_fpr <= 1:
        raise ValueError(f"Arguments `max_fpr` should be a float in range (0, 1], but got: {max_fpr}")


def _warn_degenerate(counts_row: Tensor) -> None:
    n_pos, n_neg = int(counts_row[0]), int(counts_row[1])
    if n_neg <= 0:
        rank_zero_warn(
            "No negative samples in targets, false positive value should be meaningless."
            " Returning zero tensor in false positive score",
            UserWarning,
        )
    if n_pos <= 0:
        rank_zero_warn(
            "No positive samples in targets, true positive value should be meaningless."
            " Returning zero tensor in true positive score",
            UserWarning,
        )


def _binary_auroc_compute(
    state: Union[Tensor, tuple[Tensor, Tensor]],
    thresholds: Optional[Tensor],
    max_fpr: Optional[float] = None,
    pos_label: int = 1,
    scalars: Optional[tuple] = None,
) -> Tensor:
    """Area under the ROC curve (reference :83-107).  ``scalars``: an already available ``(auroc, ap, counts)``
    evaluation of the same state (metric classes share one per compute group)."""
    if thresholds is None and (max_fpr is None or max_fpr == 1):
        if scalars is not None:
            auroc, _, counts = scalars
        else:
            preds, target = state
            if preds.numel() == 0:
                raise IndexError("metrics_b200: cannot compute AUROC from zero samples")
            auroc, _, counts, _ = _native.curve_evaluate(preds, target, 1, pos_label, want_curve=False)
        _warn_degenerate(counts[0].cpu())  # the reference branches on `fps[-1] <= 0` / `tps[-1] <= 0` (host sync) too
        return auroc[0]

    fpr, tpr, _ = _binary_roc_compute(state, thresholds, pos_label)
    if max_fpr is None or max_fpr == 1 or fpr.sum() == 0 or tpr.sum() == 0:
        return _auc_compute_without_check(fpr, tpr, 1.0)
    max_area: Tensor = tensor(max_fpr, device=fpr.device)
    # add one point at max_fpr by linear interpolation, then McClish-standardise the partial area
    stop = torch.bucketize(max_area, fpr, out_int32=True, right=True)
    weight = (max_area - fpr[stop - 1]) / (fpr[stop] - fpr[stop - 1])
    interp_tpr: Tensor = torch.lerp(tpr[stop - 1], tpr[stop], weight)
    tpr = torch.cat([tpr[:stop], interp_tpr.view(1)])
    fpr = torch.cat([fpr[:stop], max_area.view(1)])
    partial_auc = _auc_compute_without_check(fpr, tpr, 1.0)
    min_area: Tensor = 0.5 * max_area**2
    return 0.5 * (1 + (partial_auc - min_area) / (max_area - min_area))


def binary_auroc(
    preds: Tensor,
    target: Tensor,
    max_fpr: Optional[float] = None,
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
    validate_args: bool = True,
) -> Tensor:
    """Binary AUROC — reference :110-178."""
    if validate_args:
        _binary_auroc_arg_validation(max_fpr, thresholds, ignore_index)
        _binary_precision_recall_curve_tensor_validation(preds, target, ignore_index)
    preds, target, thresholds = _binary_precision_recall_curve_format(preds, target, thresholds, ignore_index)
    state = _binary_precision_recall_curve_update(preds, target, thresholds)
    return _binary_auroc_compute(state, thresholds, max_fpr)


def _multiclass_auroc_arg_validation(
    num_classes: int,
    average: Optional[str] = "macro",
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
) -> None:
    _multiclass_precision_recall_curve_arg_validation(num_classes, thresholds, ignore_index)
    allowed_average = ("macro", "weighted", "none", None)
    if average not in allowed_average:
        raise ValueError(f"Expected argument `average` to be one of {allowed_average} but got {average}")


def _multiclass_auroc_compute(
    state: Union[Tensor, tuple[Tensor, Tensor]],
    num_classes: int,
    average: Optional[str] = "macro",
    thresholds: Optional[Tensor] = None,
    scalars: Optional[tuple] = None,
) -> Tensor:
    """Per-class one-vs-rest AUROC from ONE batched sort + scan, then the class reduction (reference :193-205).
    Classes without positives (or without negatives) score 0 and ARE part of the macro mean, like the reference."""
    if isinstance(state, Tensor) and thresholds is not None:  # binned
        fpr, tpr, _ = _multiclass_roc_compute(state, num_classes, thresholds)
        res = _auc_compute_without_check(fpr, tpr, 1.0, axis=1)
        return _reduce_per_class(res, average, state[0][:, 1, :].sum(-1).float(), "Average precision")
    if scalars is not None:
        auroc, _, counts = scalars
    else:
        preds, target = state
        auroc, _, counts, _ = _native.curve_evaluate(preds, target, num_classes, want_curve=False)
    return _reduce_per_class(auroc, average, counts[:, 0].float(), "Average precision")


def multiclass_auroc(
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    average: Optional[Literal["macro", "weighted", "none"]] = "macro",
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
    validate_args: bool = True,
) -> Tensor:
    """Multiclass one-vs-rest AUROC — reference :208-300."""
    if validate_args:
        _multiclass_auroc_arg_validation(num_classes, average, thresholds, ignore_index)
        _multiclass_precision_recall_curve_tensor_validation(preds, target, num_classes, ignore_index)
    preds, target, thresholds = _multiclass_precision_recall_curve_format(
        preds, target, num_classes, thresholds, ignore_index
    )
    state = _multiclass_precision_recall_curve_update(preds, target, num_classes, thresholds)
    return _multiclass_auroc_compute(state, num_classes, average, thresholds)


# ----------------------------------------------------------------------------------------------------------------------
# multilabel (reference auroc.py:292-425)
# ----------------------------------------------------------------------------------------------------------------------
def _multilabel_auroc_arg_validation(
    num_labels: int,
    average: Optional[str],
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
) -> None:
    from metrics_b200.functional.classification.precision_recall_curve import _multilabel_precision_recall_curve_arg_validation

    _multilabel_precision_recall_curve_arg_validation(num_labels, thresholds, ignore_index)
    allowed_average = ("micro", "macro", "weighted", "none", None)
    if average not in allowed_average:
        raise ValueError(f"Expected argument `average` to be one of {allowed_average} but got {average}")


def _multilabel_micro_state(state, ignore_index: Optional[int]):
    preds, target = state[0].flatten(), state[1].flatten()
    if ignore_index is not None:
        keep = target != ignore_index
        preds, target = preds[keep], target[keep]
    return preds, target


def _multilabel_auroc_compute(
    state: Union[Tensor, tuple[Tensor, Tensor]],
    num_labels: int,
    average: Optional[str],
    thresholds: Optional[Tensor],
    ignore_index: Optional[int] = None,
    scalars: Optional[tuple] = None,
) -> Tensor:
    """Per-label AUROC from ONE batched sort + scan (reference :308-333 sorts once per label)."""
    from metrics_b200.functional.classification.roc import _multilabel_roc_compute

    if average == "micro":
        if isinstance(state, Tensor) and thresholds is not None:
            return _binary_auroc_compute(state.sum(1), thresholds, max_fpr=None)
        return _binary_auroc_compute(_multilabel_micro_state(state, ignore_index), thresholds, max_fpr=None)
    if isinstance(state, Tensor) and thresholds is not None:  # binned
        fpr, tpr, _ = _multilabel_roc_compute(state, num_labels, thresholds, ignore_index)
        res = _auc_compute_without_check(fpr, tpr, 1.0, axis=1)
        return _reduce_per_class(res, average, state[0][:, 1, :].sum(-1).float(), "Average precision")
    if scalars is not None:
        auroc, _, counts = scalars
    else:
        auroc, _, counts, _ = _native.curve_evaluate_multilabel(state[0], state[1], num_labels, ignore_index)
    return _reduce_per_class(auroc, average, counts[:, 0].float(), "Average precision")


def multilabel_auroc(
    preds: Tensor,
    target: Tensor,
    num_labels: int,
    average: Optional[Literal["micro", "macro", "weighted", "none"]] = "macro",
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
    validate_args: bool = True,
) -> Tensor:
    """Multilabel AUROC — reference :336-425."""
    from metrics_b200.functional.classification.precision_recall_curve import (
        _multilabel_precision_recall_curve_format,
        _multilabel_precision_recall_curve_tensor_validation,
        _multilabel_precision_recall_curve_update,
    )

    if validate_args:
        _multilabel_auroc_arg_validation(num_labels, average, thresholds, ignore_index)
        _multilabel_precision_recall_curve_tensor_validation(preds, target, num_labels, ignore_index)
    preds, target, thresholds = _multilabel_precision_recall_curve_format(preds, target, num_labels, thresholds, ignore_index)
    state = _multilabel_precision_recall_curve_update(preds, target, num_labels, thresholds, ignore_index)
    return _multilabel_auroc_compute(state, num_labels, average, thresholds, ignore_index)


def auroc(preds: Tensor, target: Tensor, task: Literal["binary", "multiclass", "multilabel"],
          thresholds: Optional[Union[int, List[float], Tensor]] = None, num_classes: Optional[int] = None,
          num_labels: Optional[int] = None, average: Optional[Literal["macro", "weighted", "none"]] = "macro",
          max_fpr: Optional[float] = None, ignore_index: Optional[int] = None, validate_args: bool = True) -> Optional[Tensor]:
    """Task wrapper (reference :428-491)."""
    from metrics_b200.functional.classification._task import call_for_task

    return call_for_task(
        task, num_classes, num_labels,
        lambda: binary_auroc(preds, target, max_fpr, thresholds, ignore_index, validate_args),
        lambda c: multiclass_auroc(preds, target, c, average, thresholds, ignore_index, validate_args),
        lambda n: multilabel_auroc(preds, target, n, average, thresholds, ignore_index, validate_args))
