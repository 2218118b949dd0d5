"""Mean intersection over union for semantic segmentation (reference: functional/segmentation/mean_iou.py).

The counts come from kernel K15 (`utils._overlap_counts`); the float epilogue runs in torch ops on the ``[N, C']``
counts, in the reference's op order."""
from __future__ import annotations

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200.functional.segmentation.utils import _overlap_counts
from metrics_b200.utilities.compute import _safe_divide


def _mean_iou_validate_args(
    num_classes: int,
    include_background: bool,
    per_class: bool,
    input_format: Literal["one-hot", "index"] = "one-hot",
) -> None:
    """Validate the arguments of the metric."""
    if num_classes <= 0:
        raise ValueError(f"Expected argument `num_classes` must be a positive integer, but got {num_classes}.")
    if not isinstance(include_background, bool):
        raise ValueError(f"Expected argument `include_background` must be a boolean, but got {include_background}.")
    if not isinstance(per_class, bool):
        raise ValueError(f"Expected argument `per_class` must be a boolean, but got {per_class}.")
    if input_format not in ["one-hot", "index"]:
        raise ValueError(f"Expected argument `input_format` to be one of 'one-hot', 'index', but got {input_format}.")


def _mean_iou_update(
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    include_background: bool = False,
    input_format: Literal["one-hot", "index"] = "one-hot",
) -> tuple[Tensor, Tensor]:
    """Per-sample, per-class intersection and union (int64 ``[N, C']``)."""
    intersection, pred_sum, target_sum = _overlap_counts(preds, target, num_classes, include_background, input_format, "and")
    union = target_sum + pred_sum - intersection
    return intersection, union


def _mean_iou_compute(
    intersection: Tensor,
    union: Tensor,
    per_class: bool = False,
) -> Tensor:
    """IoU per sample and class, or its mean over the classes."""
    val = _safe_divide(intersection, union)
    return val if per_class else torch.mean(val, 1)


def mean_iou(
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    include_background: bool = True,
    per_class: bool = False,
    input_format: Literal["one-hot", "index"] = "one-hot",
) -> Tensor:
    """Mean Intersection over Union (mIoU) of every sample, ``[N]``, or ``[N, C']`` with ``per_class=True``.

    ``preds`` / ``target``: one-hot ``(N, C, ...)`` integer or bool tensors, or int64 class indices ``(N, ...)`` with
    ``input_format="index"``; CUDA tensors."""
    _mean_iou_validate_args(num_classes, include_background, per_class, input_format)
    intersection, union = _mean_iou_update(preds, target, num_classes, include_background, input_format)
    return _mean_iou_compute(intersection, union, per_class=per_class)
