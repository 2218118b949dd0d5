"""Dice score for semantic segmentation (reference: functional/segmentation/dice.py).

The counts come from kernel K15 (`utils._overlap_counts`, intersection ``sum(preds * target)``); the rest runs in torch
ops on the ``[N, C']`` counts, in the reference's op order."""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200.functional.segmentation.utils import _overlap_counts
from metrics_b200.utilities.compute import _safe_divide


def _dice_score_validate_args(
    num_classes: int,
    include_background: bool,
    average: Optional[Literal["micro", "macro", "weighted", "none"]] = "micro",
    input_format: Literal["one-hot", "index"] = "one-hot",
) -> None:
    """Validate the arguments of the metric."""
    if not isinstance(num_classes, int) or num_classes <= 0:
        raise ValueError(f"Expected argument `num_classes` must be a positive integer, but got {num_classes}.")
    if not isinstance(include_background, bool):
        raise ValueError(f"Expected argument `include_background` must be a boolean, but got {include_background}.")
    allowed_average = ["micro", "macro", "weighted", "none"]
    if average is not None and average not in allowed_average:
        raise ValueError(f"Expected argument `average` to be one of {allowed_average} or None, but got {average}.")
    if input_format not in ["one-hot", "index"]:
        raise ValueError(f"Expected argument `input_format` to be one of 'one-hot', 'index', but got {input_format}.")


def _dice_score_update(
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    include_background: bool,
    input_format: Literal["one-hot", "index"] = "one-hot",
) -> tuple[Tensor, Tensor, Tensor]:
    """``(2 * intersection, pred_sum + target_sum, target_sum)``, each ``[N, C']``."""
    intersection, pred_sum, target_sum = _overlap_counts(preds, target, num_classes, include_background, input_format, "mul")
    return 2 * intersection, pred_sum + target_sum, target_sum


def _dice_score_compute(
    numerator: Tensor,
    denominator: Tensor,
    average: Optional[Literal["micro", "macro", "weighted", "none"]] = "micro",
    support: Optional[Tensor] = None,
) -> Tensor:
    """Dice score per sample from the per-class numerators and denominators."""
    if average == "micro":
        numerator = torch.sum(numerator, dim=-1)
        denominator = torch.sum(denominator, dim=-1)
    dice = _safe_divide(numerator, denominator, zero_division=1.0)
    if average == "macro":
        dice = torch.mean(dice, dim=-1)
    elif average == "weighted" and support is not None:
        weights = _safe_divide(support, torch.sum(support, dim=-1, keepdim=True), zero_division=1.0)
        dice = torch.sum(dice * weights, dim=-1)
    return dice


def dice_score(
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    include_background: bool = True,
    average: Optional[Literal["micro", "macro", "weighted", "none"]] = "micro",
    input_format: Literal["one-hot", "index"] = "one-hot",
) -> Tensor:
    """Dice score of every sample, ``[N]``, or ``[N, C']`` with ``average="none"`` / ``None``.

    ``preds`` / ``target``: one-hot ``(N, C, ...)`` tensors (bool, integer, float32 / float16 / bfloat16), or int64 class
    indices ``(N, ...)`` with ``input_format="index"``; CUDA tensors."""
    _dice_score_validate_args(num_classes, include_background, average, input_format)
    numerator, denominator, support = _dice_score_update(preds, target, num_classes, include_background, input_format)
    return _dice_score_compute(numerator, denominator, average, support=support)
