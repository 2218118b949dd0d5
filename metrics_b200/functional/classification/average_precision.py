"""Average-precision functionals, exact mode (reference: functional/classification/average_precision.py).

AP = sum over distinct thresholds of (recall_i - recall_{i-1}) * precision_i, accumulated inside the scan kernel in
fp64 (fixed order) — no precision/recall arrays are materialised.
"""
from __future__ import annotations

from typing import List, Optional, Union

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200 import _native
from metrics_b200.functional.classification.auroc import _reduce_per_class
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
from metrics_b200.functional.classification.precision_recall_curve import (  # noqa: E402
    _binary_precision_recall_curve_compute,
    _multiclass_precision_recall_curve_compute,
)
from metrics_b200.utilities.prints import rank_zero_warn


def _reduce_average_precision(res: Tensor, average: Optional[str] = "macro", weights: Optional[Tensor] = None) -> Tensor:
    return _reduce_per_class(res, average, weights, "Average precision")


def _binary_average_precision_compute(
    state: Union[Tensor, tuple[Tensor, Tensor]], thresholds: Optional[Tensor], pos_label: int = 1,
    scalars: Optional[tuple] = None,
) -> Tensor:
    """Reference :70-75.  With no positive sample the reference warns, forces recall to 1 and returns -0.0."""
    if isinstance(state, Tensor) and thresholds is not None:  # binned
        precision, recall, _ = _binary_precision_recall_curve_compute(state, thresholds)
        return -torch.sum((recall[1:] - recall[:-1]) * precision[:-1])
    preds, target = state
    if scalars is not None:
        _, ap, counts = scalars
    else:
        if preds.numel() == 0:
            raise IndexError("metrics_b200: cannot compute average precision from zero samples")
        _, ap, counts, _ = _native.curve_evaluate(preds, target, 1, pos_label, want_curve=False)
    if int(counts[0, 0]) == 0 and bool((target == 0).all()):
        rank_zero_warn(
            "No positive samples found in target, recall is undefined. Setting recall to one for all thresholds.",
            UserWarning,
        )
    return ap[0]


def binary_average_precision(
    preds: Tensor,
    target: Tensor,
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
    validate_args: bool = True,
) -> Tensor:
    """Binary average precision — reference :78-150."""
    if validate_args:
        _binary_precision_recall_curve_arg_validation(thresholds, ignore_index)
        _binary_precision_recall_curve_tensor_validation(preds, target, ignore_index)
    preds, target, thresholds = _binary_precision_recall_curve_format(preds, target, thresholds, ignore_index)
    state = _binary_precision_recall_curve_update(preds, target, thresholds)
    return _binary_average_precision_compute(state, thresholds)


def _multiclass_average_precision_arg_validation(
    num_classes: int,
    average: Optional[str] = "macro",
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
) -> None:
    _multiclass_precision_recall_curve_arg_validation(num_classes, thresholds, ignore_index)
    allowed_average = ("macro", "weighted", "none", None)
    if average not in allowed_average:
        raise ValueError(f"Expected argument `average` to be one of {allowed_average} but got {average}")


def _multiclass_average_precision_compute(
    state: Union[Tensor, tuple[Tensor, Tensor]],
    num_classes: int,
    average: Optional[str] = "macro",
    thresholds: Optional[Tensor] = None,
    scalars: Optional[tuple] = None,
) -> Tensor:
    """Per-class one-vs-rest AP from ONE batched sort + scan (reference :164-176).

    A class without positives has recall 0/0 = NaN in the reference (its all-negative guard looks at
    ``(target == 0).all()`` of the multiclass target, functional/.../precision_recall_curve.py:278), so its AP is NaN
    and it is dropped from macro/weighted means with a warning — unless every target is class 0, in which case the
    guard fires for every class and absent classes score -0.0.
    """
    if isinstance(state, Tensor) and thresholds is not None:  # binned
        precision, recall, _ = _multiclass_precision_recall_curve_compute(state, num_classes, thresholds)
        res = -torch.sum((recall[:, 1:] - recall[:, :-1]) * precision[:, :-1], 1)
        return _reduce_average_precision(res, average, weights=state[0][:, 1, :].sum(-1).float())
    preds, target = state
    if scalars is not None:
        _, ap, counts = scalars
    else:
        _, ap, counts, _ = _native.curve_evaluate(preds, target, num_classes, want_curve=False)
    n_pos = counts[:, 0]
    if not bool((target == 0).all()):
        ap = torch.where(n_pos == 0, torch.full_like(ap, float("nan")), ap)
    return _reduce_average_precision(ap, average, weights=n_pos.float())


def multiclass_average_precision(
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    average: Optional[Literal["macro", "weighted", "none"]] = "macro",
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
    validate_args: bool = True,
) -> Tensor:
    """Multiclass one-vs-rest average precision — reference :179-270."""
    if validate_args:
        _multiclass_average_precision_arg_validation(num_classes, average, thresholds, ignore_index)
        _multiclass_precision_recall_curve_tensor_validation(preds, target, num_classes, ignore_index)
    preds, target, thresholds = _multiclass_precision_recall_curve_format(
        preds, target, num_classes, thresholds, ignore_index
    )
    state = _multiclass_precision_recall_curve_update(preds, target, num_classes, thresholds)
    return _multiclass_average_precision_compute(state, num_classes, average, thresholds)


# ----------------------------------------------------------------------------------------------------------------------
# multilabel (reference average_precision.py:272-420)
# ----------------------------------------------------------------------------------------------------------------------
def _multilabel_average_precision_arg_validation(
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


def _multilabel_average_precision_compute(
    state: Union[Tensor, tuple[Tensor, Tensor]],
    num_labels: int,
    average: Optional[str],
    thresholds: Optional[Tensor],
    ignore_index: Optional[int] = None,
    scalars: Optional[tuple] = None,
) -> Tensor:
    """Per-label AP from ONE batched sort + scan (reference :284-309).  A label without positives scores -0.0 (the
    per-label binary all-negative guard), never NaN."""
    from metrics_b200.functional.classification.auroc import _multilabel_micro_state
    from metrics_b200.functional.classification.precision_recall_curve import _multilabel_precision_recall_curve_compute

    if average == "micro":
        if isinstance(state, Tensor) and thresholds is not None:
            return _binary_average_precision_compute(state.sum(1), thresholds)
        return _binary_average_precision_compute(_multilabel_micro_state(state, ignore_index), thresholds)
    if isinstance(state, Tensor) and thresholds is not None:  # binned
        precision, recall, _ = _multilabel_precision_recall_curve_compute(state, num_labels, thresholds, ignore_index)
        res = -torch.sum((recall[:, 1:] - recall[:, :-1]) * precision[:, :-1], 1)
        return _reduce_average_precision(res, average, weights=state[0][:, 1, :].sum(-1).float())
    if scalars is not None:
        _, ap, counts = scalars
    else:
        _, ap, counts, _ = _native.curve_evaluate_multilabel(state[0], state[1], num_labels, ignore_index)
    if bool((counts[:, 0] == 0).any()):
        rank_zero_warn(
            "No positive samples found in target, recall is undefined. Setting recall to one for all thresholds.",
            UserWarning,
        )
    return _reduce_average_precision(ap, average, weights=counts[:, 0].float())


def multilabel_average_precision(
    preds: Tensor,
    target: Tensor,
    num_labels: int,
    average: Optional[Literal["micro", "macro", "weighted", "none"]] = "macro",
    thresholds: Optional[Union[int, List[float], Tensor]] = None,
    ignore_index: Optional[int] = None,
    validate_args: bool = True,
) -> Tensor:
    """Multilabel average precision — reference :312-420."""
    from metrics_b200.functional.classification.precision_recall_curve import (
        _multilabel_precision_recall_curve_format,
        _multilabel_precision_recall_curve_tensor_validation,
        _multilabel_precision_recall_curve_update,
    )

    if validate_args:
        _multilabel_average_precision_arg_validation(num_labels, average, thresholds, ignore_index)
        _multilabel_precision_recall_curve_tensor_validation(preds, target, num_labels, ignore_index)
    preds, target, thresholds = _multilabel_precision_recall_curve_format(preds, target, num_labels, thresholds, ignore_index)
    state = _multilabel_precision_recall_curve_update(preds, target, num_labels, thresholds, ignore_index)
    return _multilabel_average_precision_compute(state, num_labels, average, thresholds, ignore_index)


def average_precision(preds: Tensor, target: Tensor, task: Literal["binary", "multiclass", "multilabel"],
                      thresholds: Optional[Union[int, List[float], Tensor]] = None, num_classes: Optional[int] = None,
                      num_labels: Optional[int] = None, average: Optional[Literal["macro", "weighted", "none"]] = "macro",
                      ignore_index: Optional[int] = None, validate_args: bool = True) -> Optional[Tensor]:
    """Task wrapper (reference :423-490)."""
    from metrics_b200.functional.classification._task import call_for_task

    return call_for_task(
        task, num_classes, num_labels,
        lambda: binary_average_precision(preds, target, thresholds, ignore_index, validate_args),
        lambda c: multiclass_average_precision(preds, target, c, average, thresholds, ignore_index, validate_args),
        lambda n: multilabel_average_precision(preds, target, n, average, thresholds, ignore_index, validate_args))
