"""Image metrics (reference: src/torchmetrics/image/).  Like the reference, not exported from the top-level package:
`from metrics_b200.image import StructuralSimilarityIndexMeasure`.

`VisualInformationFidelity` and `UniversalImageQualityIndex` are importable from here and from their modules but are not
listed in `__all__`, which names the structural-similarity classes only (as `HausdorffDistance` stays out of the
segmentation package's list)."""
from metrics_b200.image.ssim import MultiScaleStructuralSimilarityIndexMeasure, StructuralSimilarityIndexMeasure
from metrics_b200.image.uqi import UniversalImageQualityIndex  # noqa: F401
from metrics_b200.image.vif import VisualInformationFidelity  # noqa: F401

__all__ = ["MultiScaleStructuralSimilarityIndexMeasure", "StructuralSimilarityIndexMeasure"]
