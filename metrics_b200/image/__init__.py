"""Image metrics (reference: src/torchmetrics/image/).  Like the reference, not exported from the top-level package:
`from metrics_b200.image import StructuralSimilarityIndexMeasure`."""
from metrics_b200.image.ssim import MultiScaleStructuralSimilarityIndexMeasure, StructuralSimilarityIndexMeasure

__all__ = ["MultiScaleStructuralSimilarityIndexMeasure", "StructuralSimilarityIndexMeasure"]
