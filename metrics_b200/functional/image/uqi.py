"""Universal image quality index (reference: functional/image/uqi.py).

One call of kernel K21 (`mb200_uqi_update`): K20's windowed moments of the reflect-padded inputs, the UQI map and
float64 per-image sums over the reference's crop; ``reduction="none"`` also writes the map and returns the reference's
slice of it.  An update never synchronises the host.  Errors that follow from shapes and dtypes are raised before any
launch by the same torch call on a zero-stride stand-in (DESIGN.md K21)."""
from __future__ import annotations

from collections.abc import Sequence
from typing import Optional

import torch
from torch import Tensor
from torch.nn import functional as F  # noqa: N812
from typing_extensions import Literal

from metrics_b200 import _native
from metrics_b200.functional.image.ssim import _no_graph, _weights
from metrics_b200.utilities.checks import _check_same_shape

_NO_GRAPH = ("metrics_b200: the universal image quality index runs in CUDA kernels that record no autograd graph "
             "(is_differentiable is False), and an input requires grad: compute it under torch.no_grad() or on detached "
             "inputs")
_REDUCTIONS = ("elementwise_mean", "sum", "none", None)


def _uqi_update(preds: Tensor, target: Tensor) -> tuple[Tensor, Tensor]:
    """The reference's input checks, in its order."""
    if preds.dtype != target.dtype:
        raise TypeError(
            "Expected `preds` and `target` to have the same data type."
            f" Got preds: {preds.dtype} and target: {target.dtype}."
        )
    _check_same_shape(preds, target)
    if len(preds.shape) != 4:
        raise ValueError(
            f"Expected `preds` and `target` to have BxCxHxW shape. Got preds: {preds.shape} and target: {target.shape}."
        )
    return preds, target


def _raise_shape_errors(preds: Tensor, axes: list, pad_h: int, pad_w: int, reduction) -> None:
    """The errors the reference meets after its argument checks, in its order, raised by the same torch calls on
    zero-stride stand-ins of the shape (nothing the size of the input is allocated, nothing is launched)."""
    dtype = preds.dtype
    if not dtype.is_floating_point:
        _weights(axes, dtype, "cpu")  # bool: arange is not implemented
    b, c, h, w = preds.shape
    if preds.numel() == 0 or pad_h >= w or pad_w >= h:
        F.pad(torch.zeros((), dtype=torch.float32).expand(*preds.shape), (pad_h, pad_h, pad_w, pad_w), mode="reflect")
    if not dtype.is_floating_point:
        F.conv2d(torch.zeros((), dtype=dtype).expand(1, 1, axes[1][1], axes[2][1]),
                 torch.zeros((), dtype=torch.float32).expand(1, 1, axes[1][1], axes[2][1]))
    if h + 2 * pad_w < axes[1][1] or w + 2 * pad_h < axes[2][1]:
        F.conv2d(torch.zeros((), dtype=torch.float32).expand(1, c, h + 2 * pad_w, w + 2 * pad_h),
                 torch.zeros((), dtype=torch.float32).expand(c, 1, axes[1][1], axes[2][1]), groups=c)
    if b == 0:
        raise IndexError("tuple index out of range")
    if reduction not in _REDUCTIONS:
        raise ValueError("Reduction parameter unknown.")


def _uqi_compute(
    preds: Tensor,
    target: Tensor,
    kernel_size: Sequence[int] = (11, 11),
    sigma: Sequence[float] = (1.5, 1.5),
    reduction: Optional[Literal["elementwise_mean", "sum", "none"]] = "elementwise_mean",
) -> Tensor:
    """UQI of checked inputs, reduced, in ``preds``' dtype: one K21 call.

    The reference pads the width by ``pad_h = (kernel_size[0] - 1) // 2`` and the height by ``pad_w``, filters with
    ``kernel_size[0]`` taps along the height, and crops ``[pad_h : -pad_h, pad_w : -pad_w]``; all three carry over."""
    if len(kernel_size) != 2 or len(sigma) != 2:
        raise ValueError(
            "Expected `kernel_size` and `sigma` to have the length of two."
            f" Got kernel_size: {len(kernel_size)} and sigma: {len(sigma)}."
        )
    if any(x % 2 == 0 or x <= 0 for x in kernel_size):
        raise ValueError(f"Expected `kernel_size` to have odd positive number. Got {kernel_size}.")
    if any(y <= 0 for y in sigma):
        raise ValueError(f"Expected `sigma` to have positive number. Got {sigma}.")
    dtype = preds.dtype
    axes = [("u", 1, None), ("g", kernel_size[0], sigma[0]), ("g", kernel_size[1], sigma[1])]
    pad_h = (kernel_size[0] - 1) // 2
    pad_w = (kernel_size[1] - 1) // 2
    _raise_shape_errors(preds, axes, pad_h, pad_w, reduction)
    weights = _weights(axes, dtype, preds.device)
    want_map = reduction not in ("elementwise_mean", "sum")
    sums, img = _native.uqi(preds, target, weights, (1, kernel_size[0], kernel_size[1]), (0, pad_w, pad_h),
                            (pad_h, pad_w), torch.finfo(dtype).eps, want_map)
    if want_map:
        return img.squeeze(2)[..., pad_h:-pad_h, pad_w:-pad_w]
    total = sums.sum()
    if reduction == "sum":
        return total.to(dtype)
    b, c, oh, ow = (*preds.shape[:2], *_out_size(preds.shape[2:], kernel_size, pad_h, pad_w))
    count = b * c * len(range(oh)[pad_h:-pad_h]) * len(range(ow)[pad_w:-pad_w])
    return (total / count).to(dtype)  # an empty crop: 0 / 0, NaN, as the mean of an empty tensor


def _out_size(spatial, kernel_size, pad_h: int, pad_w: int) -> tuple[int, int]:
    """Output height and width of the padded, filtered image."""
    return spatial[0] + 2 * pad_w - kernel_size[0] + 1, spatial[1] + 2 * pad_h - kernel_size[1] + 1


def universal_image_quality_index(
    preds: Tensor,
    target: Tensor,
    kernel_size: Sequence[int] = (11, 11),
    sigma: Sequence[float] = (1.5, 1.5),
    reduction: Optional[Literal["elementwise_mean", "sum", "none"]] = "elementwise_mean",
) -> Tensor:
    """Universal image quality index of CUDA ``[B, C, H, W]`` float tensors (reference :119-171).  Same arguments,
    results and errors as the reference.  Moments are taken about a local shift; float16 / bfloat16 are computed in
    float32 and rounded once.  Raises ``RuntimeError`` when grad mode is on and an input requires grad."""
    preds, target = _uqi_update(preds, target)
    _no_graph(preds, target, _NO_GRAPH)
    return _uqi_compute(preds, target, kernel_size, sigma, reduction)
