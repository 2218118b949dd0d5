"""Generalized dice score for semantic segmentation (reference: functional/segmentation/generalized_dice.py).

The counts come from kernel K15 (`utils._overlap_counts`, intersection ``sum(preds * target)``); the class weights and the
rest run in torch ops on the ``[N, C']`` counts, in the reference's op order."""
from __future__ import annotations

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200.functional.segmentation.utils import _overlap_counts
from metrics_b200.utilities.compute import _safe_divide


def _generalized_dice_validate_args(
    num_classes: int,
    include_background: bool,
    per_class: bool,
    weight_type: Literal["square", "simple", "linear"],
    input_format: Literal["one-hot", "index"],
) -> None:
    """Validate the arguments of the metric."""
    if not isinstance(num_classes, int) or num_classes <= 0:
        raise ValueError(f"Expected argument `num_classes` must be a positive integer, but got {num_classes}.")
    if not isinstance(include_background, bool):
        raise ValueError(f"Expected argument `include_background` must be a boolean, but got {include_background}.")
    if not isinstance(per_class, bool):
        raise ValueError(f"Expected argument `per_class` must be a boolean, but got {per_class}.")
    if weight_type not in ["square", "simple", "linear"]:
        raise ValueError(
            f"Expected argument `weight_type` to be one of 'square', 'simple', 'linear', but got {weight_type}."
        )
    if input_format not in ["one-hot", "index"]:
        raise ValueError(f"Expected argument `input_format` to be one of 'one-hot', 'index', but got {input_format}.")


def _fill_infinite_weights(weights: Tensor) -> Tensor:
    """Replace the infinite weights of classes absent from a sample's target with the values the reference gives them
    (functional/segmentation/generalized_dice.py:84-90).  There the flat view shares storage with ``weights``, so the
    infinities are zeroed before the per-class maxima are taken, and flat element ``i`` takes the maximum of class
    ``i // N`` (the class maxima repeated N times, transposed and flattened), not the maximum of its own class.  Written
    with ``masked_fill`` / ``where`` instead of boolean-index assignment: same values, no host synchronisation."""
    n = weights.shape[0]
    flat = weights.flatten()
    absent = torch.isinf(flat)
    flat = flat.masked_fill(absent, 0)
    class_max = torch.max(flat.reshape(weights.shape), 0).values
    by_flat_index = class_max.repeat(n, 1).T.flatten()
    return torch.where(absent, by_flat_index, flat).reshape(weights.shape)


def _generalized_dice_update(
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    include_background: bool,
    weight_type: Literal["square", "simple", "linear"] = "square",
    input_format: Literal["one-hot", "index"] = "one-hot",
) -> tuple[Tensor, Tensor]:
    """Weighted numerators ``2 * intersection * w`` and denominators ``(target_sum + pred_sum) * w``, each ``[N, C']``."""
    intersection, pred_sum, target_sum = _overlap_counts(preds, target, num_classes, include_background, input_format, "mul")
    cardinality = target_sum + pred_sum
    if weight_type == "simple":
        weights = 1.0 / target_sum
    elif weight_type == "linear":
        weights = torch.ones_like(target_sum)
    elif weight_type == "square":
        weights = 1.0 / (target_sum**2)
    else:
        raise ValueError(
            f"Expected argument `weight_type` to be one of 'simple', 'linear', 'square', but got {weight_type}."
        )
    weights = _fill_infinite_weights(weights)
    numerator = 2.0 * intersection * weights
    denominator = cardinality * weights
    return numerator, denominator


def _generalized_dice_compute(numerator: Tensor, denominator: Tensor, per_class: bool = True) -> Tensor:
    """Generalized dice score per sample (and class, with ``per_class``)."""
    if not per_class:
        numerator = torch.sum(numerator, 1)
        denominator = torch.sum(denominator, 1)
    return _safe_divide(numerator, denominator)


def generalized_dice_score(
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    include_background: bool = True,
    per_class: bool = False,
    weight_type: Literal["square", "simple", "linear"] = "square",
    input_format: Literal["one-hot", "index"] = "one-hot",
) -> Tensor:
    """Generalized dice score of every sample, ``[N]``, or ``[N, C']`` with ``per_class=True``.

    ``preds`` / ``target``: one-hot ``(N, C, ...)`` tensors (bool, integer, float32 / float16 / bfloat16), or int64 class
    indices ``(N, ...)`` with ``input_format="index"``; CUDA tensors."""
    _generalized_dice_validate_args(num_classes, include_background, per_class, weight_type, input_format)
    numerator, denominator = _generalized_dice_update(
        preds, target, num_classes, include_background, weight_type, input_format
    )
    return _generalized_dice_compute(numerator, denominator, per_class)
