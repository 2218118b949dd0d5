"""Generalized dice score, modular (reference: segmentation/generalized_dice.py)."""
from typing import Any

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200.functional.segmentation.generalized_dice import (
    _generalized_dice_compute,
    _generalized_dice_update,
    _generalized_dice_validate_args,
)
from metrics_b200.metric import Metric


class GeneralizedDiceScore(Metric):
    r"""Generalized dice score for semantic segmentation (reference :34-148).

    ``preds`` / ``target``: one-hot ``(N, C, ...)`` tensors (bool, integer, float32 / float16 / bfloat16), or int64 class
    indices ``(N, ...)`` with ``input_format="index"``.  Class weights are ``1 / target_sum**2`` (``"square"``),
    ``1 / target_sum`` (``"simple"``) or 1 (``"linear"``).  Each update adds the per-sample scores to ``score`` and the
    batch size to ``samples``; ``compute`` returns their ratio.  The counts of an update come from one read of the inputs
    (kernel K15)."""

    score: Tensor
    samples: Tensor
    full_state_update: bool = False
    is_differentiable: bool = False
    higher_is_better: bool = True
    plot_lower_bound: float = 0.0
    plot_upper_bound: float = 1.0

    def __init__(
        self,
        num_classes: int,
        include_background: bool = True,
        per_class: bool = False,
        weight_type: Literal["square", "simple", "linear"] = "square",
        input_format: Literal["one-hot", "index"] = "one-hot",
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        _generalized_dice_validate_args(num_classes, include_background, per_class, weight_type, input_format)
        self.num_classes = num_classes
        self.include_background = include_background
        self.per_class = per_class
        self.weight_type = weight_type
        self.input_format = input_format

        num_classes = num_classes - 1 if not include_background else num_classes
        self.add_state("score", default=torch.zeros(num_classes if per_class else 1), dist_reduce_fx="sum")
        self.add_state("samples", default=torch.zeros(1), dist_reduce_fx="sum")

    def update(self, preds: Tensor, target: Tensor) -> None:
        """Update the state with new data."""
        numerator, denominator = _generalized_dice_update(
            preds, target, self.num_classes, self.include_background, self.weight_type, self.input_format
        )
        self.score += _generalized_dice_compute(numerator, denominator, self.per_class).sum(dim=0)
        self.samples += preds.shape[0]

    def compute(self) -> Tensor:
        """Compute the final generalized dice score."""
        return self.score / self.samples
