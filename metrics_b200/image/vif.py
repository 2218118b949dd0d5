"""Pixel-domain visual information fidelity, modular (reference: image/vif.py).  Every update is K21
(functional/image/vif.py) with no host synchronisation; the states and the result are the reference's."""
from typing import Any

import torch
from torch import Tensor

from metrics_b200.functional.image.ssim import _no_graph
from metrics_b200.functional.image.vif import _NO_GRAPH, _vif_per_channel
from metrics_b200.metric import Metric


class VisualInformationFidelity(Metric):
    """VIF-P of CUDA ``[N, C, H, W]`` float batches (reference :23-82).

    ``vif_score`` holds the sum over images of their VIF-P (the mean over channels when ``C > 1``), ``total`` the image
    count.  Like the reference, the class does not check for 41 x 41; an image too small for some scale raises the
    reference's convolution error.  ``is_differentiable`` is False: the kernels record no autograd graph, so ``forward``
    raises when an input requires grad (``update`` never does)."""

    is_differentiable = False
    higher_is_better = True
    full_state_update = False

    vif_score: Tensor
    total: Tensor

    def __init__(self, sigma_n_sq: float = 2.0, **kwargs: Any) -> None:
        super().__init__(**kwargs)

        if not isinstance(sigma_n_sq, float) and not isinstance(sigma_n_sq, int):
            raise ValueError(f"Argument `sigma_n_sq` is expected to be a positive float or int, but got {sigma_n_sq}")

        if sigma_n_sq < 0:
            raise ValueError(f"Argument `sigma_n_sq` is expected to be a positive float or int, but got {sigma_n_sq}")

        self.add_state("vif_score", default=torch.tensor(0.0), dist_reduce_fx="sum")
        self.add_state("total", default=torch.tensor(0.0), dist_reduce_fx="sum")
        self.sigma_n_sq = sigma_n_sq

    def update(self, preds: Tensor, target: Tensor) -> None:
        """Update state with predictions and targets."""
        _no_graph(preds, target, _NO_GRAPH)
        per_channel = _vif_per_channel(preds, target, self.sigma_n_sq)  # [N, C]
        vif = per_channel.mean(1) if preds.size(1) > 1 else per_channel[:, 0]
        self.vif_score += torch.sum(vif)
        self.total += preds.shape[0]

    def compute(self) -> Tensor:
        """Compute vif-p over state."""
        return self.vif_score / self.total
