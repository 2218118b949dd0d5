"""Segmentation metrics (reference: src/torchmetrics/segmentation/).  Like the reference, not exported from the top-level
package: `from metrics_b200.segmentation import MeanIoU`.  `HausdorffDistance` is importable from here but not yet listed
in `__all__`."""
from metrics_b200.segmentation.dice import DiceScore
from metrics_b200.segmentation.generalized_dice import GeneralizedDiceScore
from metrics_b200.segmentation.hausdorff_distance import HausdorffDistance  # noqa: F401
from metrics_b200.segmentation.mean_iou import MeanIoU

__all__ = ["DiceScore", "GeneralizedDiceScore", "MeanIoU"]
