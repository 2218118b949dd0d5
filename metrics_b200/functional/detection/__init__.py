"""Functional detection metrics (reference: src/torchmetrics/functional/detection/): the panoptic qualities.  The box-IoU
family is out of scope (DESIGN.md section 0)."""
from metrics_b200.functional.detection.panoptic_qualities import modified_panoptic_quality, panoptic_quality

__all__ = ["modified_panoptic_quality", "panoptic_quality"]
