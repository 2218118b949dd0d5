"""Universal image quality index, modular (reference: image/uqi.py).  Every update is K21 (functional/image/uqi.py)
with no host synchronisation; the states, reductions and return shapes are the reference's."""
from collections.abc import Sequence
from typing import Any, List

from torch import Tensor, tensor
from typing_extensions import Literal

from metrics_b200.functional.image.ssim import _no_graph
from metrics_b200.functional.image.uqi import _NO_GRAPH, _uqi_compute, _uqi_update
from metrics_b200.metric import Metric
from metrics_b200.utilities import rank_zero_warn
from metrics_b200.utilities.data import dim_zero_cat


class UniversalImageQualityIndex(Metric):
    """Universal image quality index of CUDA ``[B, C, H, W]`` float batches (reference :31-124).

    ``"elementwise_mean"`` / ``"sum"``: ``sum_uqi`` holds the sum of the cropped maps, ``numel`` the reference's count
    ``B · C · (H − k0 + 1) · (W − k1 + 1)``, which is not the crop's size for an anisotropic ``kernel_size``.
    ``"none"`` / None: the batches are kept and the map of all of them is returned.  ``is_differentiable`` is False, as
    for StructuralSimilarityIndexMeasure."""

    is_differentiable: bool = False
    higher_is_better: bool = True
    full_state_update: bool = False
    plot_lower_bound: float = 0.0
    plot_upper_bound: float = 1.0

    preds: List[Tensor]
    target: List[Tensor]
    sum_uqi: Tensor
    numel: Tensor

    def __init__(
        self,
        kernel_size: Sequence[int] = (11, 11),
        sigma: Sequence[float] = (1.5, 1.5),
        reduction: Literal["elementwise_mean", "sum", "none", None] = "elementwise_mean",
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        if reduction not in ("elementwise_mean", "sum", "none", None):
            raise ValueError(
                f"The `reduction` {reduction} is not valid. Valid options are `elementwise_mean`, `sum`, `none`, None."
            )
        if reduction is None or reduction == "none":
            rank_zero_warn(
                "Metric `UniversalImageQualityIndex` will save all targets and predictions in the buffer when using"
                "`reduction=None` or `reduction='none'. For large datasets, this may lead to a large memory footprint."
            )
            self.add_state("preds", default=[], dist_reduce_fx="cat")
            self.add_state("target", default=[], dist_reduce_fx="cat")
        else:
            self.add_state("sum_uqi", tensor(0.0), dist_reduce_fx="sum")
            self.add_state("numel", tensor(0), dist_reduce_fx="sum")
        self.kernel_size = kernel_size
        self.sigma = sigma
        self.reduction = reduction

    def update(self, preds: Tensor, target: Tensor) -> None:
        """Update state with predictions and targets."""
        preds, target = _uqi_update(preds, target)
        _no_graph(preds, target, _NO_GRAPH)
        if self.reduction is None or self.reduction == "none":
            self.preds.append(preds)
            self.target.append(target)
        else:
            uqi_score = _uqi_compute(preds, target, self.kernel_size, self.sigma, reduction="sum")
            self.sum_uqi += uqi_score
            ps = preds.shape
            self.numel += ps[0] * ps[1] * (ps[2] - self.kernel_size[0] + 1) * (ps[3] - self.kernel_size[1] + 1)

    def compute(self) -> Tensor:
        """Compute explained variance over state."""
        if self.reduction == "none" or self.reduction is None:
            preds = dim_zero_cat(self.preds)
            target = dim_zero_cat(self.target)
            return _uqi_compute(preds, target, self.kernel_size, self.sigma, self.reduction)
        return self.sum_uqi / self.numel if self.reduction == "elementwise_mean" else self.sum_uqi
