"""Functional image metrics (reference: src/torchmetrics/functional/image/): structural similarity and its multi-scale
form, visual information fidelity and the universal image quality index.  Like the reference, not exported from the
top-level package.

`visual_information_fidelity` and `universal_image_quality_index` are importable from here and from their modules but
are not listed in `__all__`, which names the structural-similarity functionals only (as `hausdorff_distance` stays out
of the segmentation package's list)."""
from metrics_b200.functional.image.ssim import (
    multiscale_structural_similarity_index_measure,
    structural_similarity_index_measure,
)
from metrics_b200.functional.image.uqi import universal_image_quality_index  # noqa: F401
from metrics_b200.functional.image.vif import visual_information_fidelity  # noqa: F401

__all__ = ["multiscale_structural_similarity_index_measure", "structural_similarity_index_measure"]
