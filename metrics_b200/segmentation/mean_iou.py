"""Mean intersection over union, modular (reference: segmentation/mean_iou.py)."""
from typing import Any

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200.functional.segmentation.mean_iou import _mean_iou_compute, _mean_iou_update, _mean_iou_validate_args
from metrics_b200.metric import Metric


class MeanIoU(Metric):
    """Mean Intersection over Union (mIoU) for semantic segmentation (reference :30-128).

    ``preds`` / ``target``: one-hot ``(N, C, ...)`` bool or integer tensors, or int64 class indices ``(N, ...)`` with
    ``input_format="index"``.  Each update adds the batch mean of the per-sample mIoU (per class with ``per_class=True``)
    to ``score``; ``compute`` returns ``score / num_batches``.  The counts of an update come from one read of the inputs
    (kernel K15)."""

    score: Tensor
    num_batches: Tensor
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
        input_format: Literal["one-hot", "index"] = "one-hot",
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        _mean_iou_validate_args(num_classes, include_background, per_class, input_format)
        self.num_classes = num_classes
        self.include_background = include_background
        self.per_class = per_class
        self.input_format = input_format

        num_classes = num_classes - 1 if not include_background else num_classes
        self.add_state("score", default=torch.zeros(num_classes if per_class else 1), dist_reduce_fx="sum")
        self.add_state("num_batches", default=torch.tensor(0), dist_reduce_fx="sum")

    def update(self, preds: Tensor, target: Tensor) -> None:
        """Update the state with the new data."""
        intersection, union = _mean_iou_update(
            preds, target, self.num_classes, self.include_background, self.input_format
        )
        score = _mean_iou_compute(intersection, union, per_class=self.per_class)
        self.score += score.mean(0) if self.per_class else score.mean()
        self.num_batches += 1

    def compute(self) -> Tensor:
        """Compute the final Mean Intersection over Union (mIoU)."""
        return self.score / self.num_batches
