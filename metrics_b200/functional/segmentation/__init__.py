"""Functional segmentation metrics (reference: src/torchmetrics/functional/segmentation/).  `hausdorff_distance` is
importable from here but not yet listed in `__all__`."""
from metrics_b200.functional.segmentation.dice import dice_score
from metrics_b200.functional.segmentation.generalized_dice import generalized_dice_score
from metrics_b200.functional.segmentation.hausdorff_distance import hausdorff_distance  # noqa: F401
from metrics_b200.functional.segmentation.mean_iou import mean_iou

__all__ = ["dice_score", "generalized_dice_score", "mean_iou"]
