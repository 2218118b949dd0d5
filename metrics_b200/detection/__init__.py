"""Detection metrics (reference: src/torchmetrics/detection/)."""
from metrics_b200.detection.mean_ap import MeanAveragePrecision  # noqa: F401
from metrics_b200.detection.panoptic_qualities import ModifiedPanopticQuality, PanopticQuality  # noqa: F401
