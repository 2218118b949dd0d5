"""Functional image metrics (reference: src/torchmetrics/functional/image/): structural similarity and its multi-scale
form.  Like the reference, not exported from the top-level package."""
from metrics_b200.functional.image.ssim import (
    multiscale_structural_similarity_index_measure,
    structural_similarity_index_measure,
)

__all__ = ["multiscale_structural_similarity_index_measure", "structural_similarity_index_measure"]
