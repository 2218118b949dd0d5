"""Hausdorff distance, modular (reference: segmentation/hausdorff_distance.py)."""
from typing import Any, Optional, Union

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200.functional.segmentation.hausdorff_distance import (
    _hausdorff_distance_validate_args,
    hausdorff_distance,
)
from metrics_b200.metric import Metric


class HausdorffDistance(Metric):
    """Hausdorff distance between the edges of predicted and target masks for semantic segmentation (reference :31-127).

    ``preds`` / ``target``: one-hot ``(N, C, H, W)`` bool or integer tensors, or int64 class indices ``(N, H, W)`` with
    ``input_format="index"``.  Each update adds the sum of its ``[N, C']`` distances to ``score`` and their count to
    ``total``; ``compute`` returns ``score / total``.  The distances of an update come from kernel K19 (one host
    synchronisation, for its error word)."""

    is_differentiable: bool = True
    higher_is_better: bool = False
    full_state_update: bool = False
    plot_lower_bound: float = 0.0

    score: Tensor
    total: Tensor

    def __init__(
        self,
        num_classes: int,
        include_background: bool = False,
        distance_metric: Literal["euclidean", "chessboard", "taxicab"] = "euclidean",
        spacing: Optional[Union[Tensor, list[float]]] = None,
        directed: bool = False,
        input_format: Literal["one-hot", "index"] = "one-hot",
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        _hausdorff_distance_validate_args(
            num_classes, include_background, distance_metric, spacing, directed, input_format
        )
        self.num_classes = num_classes
        self.include_background = include_background
        self.distance_metric = distance_metric
        self.spacing = spacing
        self.directed = directed
        self.input_format = input_format
        self.add_state("score", default=torch.tensor(0.0), dist_reduce_fx="sum")
        self.add_state("total", default=torch.tensor(0), dist_reduce_fx="sum")

    def update(self, preds: Tensor, target: Tensor) -> None:
        """Update state with predictions and targets."""
        score = hausdorff_distance(
            preds,
            target,
            self.num_classes,
            include_background=self.include_background,
            distance_metric=self.distance_metric,
            spacing=self.spacing,
            directed=self.directed,
            input_format=self.input_format,
        )
        self.score += score.sum()
        self.total += score.numel()

    def compute(self) -> Tensor:
        """Compute final Hausdorff distance over states."""
        return self.score / self.total
