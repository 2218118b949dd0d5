"""Segmentation metrics (reference: src/torchmetrics/segmentation/), the count-based three.  `HausdorffDistance` needs
distance transforms and is out of scope (DESIGN.md section 0).  Like the reference, not exported from the top-level
package: `from metrics_b200.segmentation import MeanIoU`."""
from metrics_b200.segmentation.dice import DiceScore
from metrics_b200.segmentation.generalized_dice import GeneralizedDiceScore
from metrics_b200.segmentation.mean_iou import MeanIoU

__all__ = ["DiceScore", "GeneralizedDiceScore", "MeanIoU"]
