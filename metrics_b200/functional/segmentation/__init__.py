"""Functional segmentation metrics (reference: src/torchmetrics/functional/segmentation/), the count-based three.
`hausdorff_distance` needs distance transforms and is out of scope (DESIGN.md section 0)."""
from metrics_b200.functional.segmentation.dice import dice_score
from metrics_b200.functional.segmentation.generalized_dice import generalized_dice_score
from metrics_b200.functional.segmentation.mean_iou import mean_iou

__all__ = ["dice_score", "generalized_dice_score", "mean_iou"]
