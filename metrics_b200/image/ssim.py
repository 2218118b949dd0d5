"""Structural similarity, modular (reference: image/ssim.py).  Every update is K20 (functional/image/ssim.py) with no
host synchronisation; the states, reductions and return shapes are the reference's."""
from collections.abc import Sequence
from typing import Any, List, Optional, Union

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200.functional.image.ssim import (
    _check_msssim_args,
    _multiscale_ssim_update,
    _no_graph,
    _ssim_check_inputs,
    _ssim_update,
)
from metrics_b200.metric import Metric
from metrics_b200.utilities.data import dim_zero_cat

_VALID_REDUCTION = ("elementwise_mean", "sum", "none", None)


class StructuralSimilarityIndexMeasure(Metric):
    """Structural similarity of CUDA ``[B, C, H, W]`` or ``[B, C, D, H, W]`` float batches (reference :31-219).

    ``similarity`` holds the sum of the per-image values (``"elementwise_mean"``, ``"sum"``) or their list, ``total``
    the image count, ``image_return`` the maps or per-image contrast terms when asked.  ``is_differentiable`` is False:
    the kernel records no autograd graph, so ``forward`` raises when an input requires grad (``update`` never does)."""

    higher_is_better: bool = True
    is_differentiable: bool = False
    full_state_update: bool = False
    plot_lower_bound: float = 0.0
    plot_upper_bound: float = 1.0

    preds: List[Tensor]
    target: List[Tensor]

    def __init__(
        self,
        gaussian_kernel: bool = True,
        sigma: Union[float, Sequence[float]] = 1.5,
        kernel_size: Union[int, Sequence[int]] = 11,
        reduction: Literal["elementwise_mean", "sum", "none", None] = "elementwise_mean",
        data_range: Optional[Union[float, tuple[float, float]]] = None,
        k1: float = 0.01,
        k2: float = 0.03,
        return_full_image: bool = False,
        return_contrast_sensitivity: bool = False,
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        if reduction not in _VALID_REDUCTION:
            raise ValueError(f"Argument `reduction` must be one of {_VALID_REDUCTION}, but got {reduction}")
        if reduction in ("elementwise_mean", "sum"):
            self.add_state("similarity", default=torch.tensor(0.0), dist_reduce_fx="sum")
        else:
            self.add_state("similarity", default=[], dist_reduce_fx="cat")
        self.add_state("total", default=torch.tensor(0.0), dist_reduce_fx="sum")
        if return_contrast_sensitivity or return_full_image:
            self.add_state("image_return", default=[], dist_reduce_fx="cat")
        self.gaussian_kernel = gaussian_kernel
        self.sigma = sigma
        self.kernel_size = kernel_size
        self.reduction = reduction
        self.data_range = data_range
        self.k1 = k1
        self.k2 = k2
        self.return_full_image = return_full_image
        self.return_contrast_sensitivity = return_contrast_sensitivity

    def update(self, preds: Tensor, target: Tensor) -> None:
        """Update state with predictions and targets."""
        preds, target = _ssim_check_inputs(preds, target)
        _no_graph(preds, target)
        similarity_pack = _ssim_update(preds, target, self.gaussian_kernel, self.sigma, self.kernel_size,
                                       self.data_range, self.k1, self.k2, self.return_full_image,
                                       self.return_contrast_sensitivity)
        if isinstance(similarity_pack, tuple):
            similarity, image = similarity_pack
            self.image_return.append(image)
        else:
            similarity = similarity_pack
        if self.reduction in ("elementwise_mean", "sum"):
            self.similarity += similarity.sum()
            self.total += preds.shape[0]
        else:
            self.similarity.append(similarity)

    def compute(self) -> Union[Tensor, tuple[Tensor, Tensor]]:
        """Compute SSIM over state."""
        if self.reduction == "elementwise_mean":
            similarity = self.similarity / self.total
        elif self.reduction == "sum":
            similarity = self.similarity
        else:
            similarity = dim_zero_cat(self.similarity)
        if self.return_contrast_sensitivity or self.return_full_image:
            return similarity, dim_zero_cat(self.image_return)
        return similarity


class MultiScaleStructuralSimilarityIndexMeasure(Metric):
    """Multi-scale structural similarity of CUDA float batches (reference :221-420): K20 per scale, a pool kernel
    between scales, the ``relu`` / ``simple`` / ``** betas`` / ``prod`` epilogue as torch ops.  ``is_differentiable``
    is False, as for StructuralSimilarityIndexMeasure."""

    higher_is_better: bool = True
    is_differentiable: bool = False
    full_state_update: bool = False
    plot_lower_bound: float = 0.0
    plot_upper_bound: float = 1.0

    preds: List[Tensor]
    target: List[Tensor]

    def __init__(
        self,
        gaussian_kernel: bool = True,
        kernel_size: Union[int, Sequence[int]] = 11,
        sigma: Union[float, Sequence[float]] = 1.5,
        reduction: Literal["elementwise_mean", "sum", "none", None] = "elementwise_mean",
        data_range: Optional[Union[float, tuple[float, float]]] = None,
        k1: float = 0.01,
        k2: float = 0.03,
        betas: tuple[float, ...] = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333),
        normalize: Literal["relu", "simple", None] = "relu",
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        if reduction not in _VALID_REDUCTION:
            raise ValueError(f"Argument `reduction` must be one of {_VALID_REDUCTION}, but got {reduction}")
        if reduction in ("elementwise_mean", "sum"):
            self.add_state("similarity", default=torch.tensor(0.0), dist_reduce_fx="sum")
        else:
            self.add_state("similarity", default=[], dist_reduce_fx="cat")
        self.add_state("total", default=torch.tensor(0.0), dist_reduce_fx="sum")
        if not (isinstance(kernel_size, (Sequence, int))):
            raise ValueError(
                f"Argument `kernel_size` expected to be an sequence or an int, or a single int. Got {kernel_size}"
            )
        if isinstance(kernel_size, Sequence) and (
            len(kernel_size) not in (2, 3) or not all(isinstance(ks, int) for ks in kernel_size)
        ):
            raise ValueError(
                "Argument `kernel_size` expected to be an sequence of size 2 or 3 where each element is an int, "
                f"or a single int. Got {kernel_size}"
            )
        self.gaussian_kernel = gaussian_kernel
        self.sigma = sigma
        self.kernel_size = kernel_size
        self.reduction = reduction
        self.data_range = data_range
        self.k1 = k1
        self.k2 = k2
        _check_msssim_args(betas, None)
        self.betas = betas
        _check_msssim_args(betas, normalize)
        self.normalize = normalize

    def update(self, preds: Tensor, target: Tensor) -> None:
        """Update state with predictions and targets."""
        preds, target = _ssim_check_inputs(preds, target)
        _no_graph(preds, target)
        similarity = _multiscale_ssim_update(preds, target, self.gaussian_kernel, self.sigma, self.kernel_size,
                                             self.data_range, self.k1, self.k2, self.betas, self.normalize)
        if self.reduction in ("none", None):
            self.similarity.append(similarity)
        else:
            self.similarity += similarity.sum()
        self.total += preds.shape[0]

    def compute(self) -> Tensor:
        """Compute MS-SSIM over state."""
        if self.reduction in ("none", None):
            return dim_zero_cat(self.similarity)
        if self.reduction == "sum":
            return self.similarity
        return self.similarity / self.total
