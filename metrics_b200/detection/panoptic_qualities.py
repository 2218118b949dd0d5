"""Panoptic quality and modified panoptic quality, modular (reference: detection/panoptic_qualities.py)."""
from __future__ import annotations

from collections.abc import Collection
from typing import Any

import torch
from torch import Tensor

from metrics_b200 import _native
from metrics_b200.functional.detection._panoptic_quality_common import (
    _get_category_id_to_continuous_id,
    _get_void_color,
    _panoptic_quality_compute,
    _panoptic_quality_output,
    _panoptic_quality_update,
    _parse_categories,
    _validate_inputs,
)
from metrics_b200.metric import Metric


class _PanopticBase(Metric):
    is_differentiable: bool = False
    higher_is_better: bool = True
    full_state_update: bool = False
    plot_lower_bound: float = 0.0
    plot_upper_bound: float = 1.0

    iou_sum: Tensor
    true_positives: Tensor
    false_positives: Tensor
    false_negatives: Tensor

    _modified = False

    def _setup(self, things: Collection[int], stuffs: Collection[int], allow_unknown_preds_category: bool) -> None:
        things, stuffs = _parse_categories(things, stuffs)
        self.things = things
        self.stuffs = stuffs
        self.void_color = _get_void_color(things, stuffs)
        self.cat_id_to_continuous_id = _get_category_id_to_continuous_id(things, stuffs)
        self.allow_unknown_preds_category = allow_unknown_preds_category
        self._categories: dict = {}  # K18's category table, per device

        num_categories = len(things) + len(stuffs)
        self.add_state("iou_sum", default=torch.zeros(num_categories, dtype=torch.double), dist_reduce_fx="sum")
        self.add_state("true_positives", default=torch.zeros(num_categories, dtype=torch.int), dist_reduce_fx="sum")
        self.add_state("false_positives", default=torch.zeros(num_categories, dtype=torch.int), dist_reduce_fx="sum")
        self.add_state("false_negatives", default=torch.zeros(num_categories, dtype=torch.int), dist_reduce_fx="sum")

    def update(self, preds: Tensor, target: Tensor) -> None:
        """Add a batch of ``(B, *spatial_dims, 2)`` integer ``(category_id, instance_id)`` maps (kernel K18)."""
        _validate_inputs(preds, target)
        categories = self._categories.get(preds.device)
        if categories is None and preds.is_cuda:
            categories = self._categories[preds.device] = _native.panoptic_categories(self.things, self.stuffs, preds.device)
        states = (self.iou_sum, self.true_positives, self.false_positives, self.false_negatives)
        _panoptic_quality_update(preds, target, self.things, self.stuffs, self.allow_unknown_preds_category, states,
                                 modified=self._modified, categories=categories)


class PanopticQuality(_PanopticBase):
    r"""`Panoptic Quality`_ :math:`PQ = \frac{IOU}{TP + 0.5 FP + 0.5 FN}` for panoptic segmentations (reference :37-290).

    ``update(preds, target)``: integer CUDA tensors ``(B, *spatial_dims, 2)`` of ``(category_id, instance_id)`` pairs.
    ``compute()``: the class average (float64 scalar); ``[pq, sq, rq]`` with ``return_sq_and_rq``; ``[1, K]`` with
    ``return_per_class``; ``[K, 3]`` with both.  Classes are the sorted things, then the sorted stuffs."""

    def __init__(
        self,
        things: Collection[int],
        stuffs: Collection[int],
        allow_unknown_preds_category: bool = False,
        return_sq_and_rq: bool = False,
        return_per_class: bool = False,
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        self._setup(things, stuffs, allow_unknown_preds_category)
        self.return_sq_and_rq = return_sq_and_rq
        self.return_per_class = return_per_class

    def update(self, preds: Tensor, target: Tensor) -> None:
        """Add a batch of ``(B, *spatial_dims, 2)`` integer ``(category_id, instance_id)`` maps (kernel K18)."""
        super().update(preds, target)

    def compute(self) -> Tensor:
        """Panoptic quality of everything passed to ``update``."""
        return _panoptic_quality_output(
            *_panoptic_quality_compute(self.iou_sum, self.true_positives, self.false_positives, self.false_negatives),
            self.return_sq_and_rq, self.return_per_class,
        )


class ModifiedPanopticQuality(_PanopticBase):
    r"""`Modified Panoptic Quality`_ for panoptic segmentations (reference :293-476): panoptic quality where a stuff class
    scores :math:`\frac{IOU_c}{|S_c|}`, the IoU sum of its overlapping segments over its number of target segments.
    ``compute()`` returns the class average (float64 scalar)."""

    _modified = True

    def __init__(
        self,
        things: Collection[int],
        stuffs: Collection[int],
        allow_unknown_preds_category: bool = False,
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        self._setup(things, stuffs, allow_unknown_preds_category)

    def update(self, preds: Tensor, target: Tensor) -> None:
        """Add a batch of ``(B, *spatial_dims, 2)`` integer ``(category_id, instance_id)`` maps (kernel K18)."""
        super().update(preds, target)

    def compute(self) -> Tensor:
        """Modified panoptic quality of everything passed to ``update``."""
        return _panoptic_quality_compute(self.iou_sum, self.true_positives, self.false_positives, self.false_negatives)[3]
