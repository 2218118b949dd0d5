"""Structural similarity and its multi-scale form (reference: functional/image/ssim.py).

Each scale is one call of kernel K20: one read of ``preds`` and ``target`` through their strides, the windowed moments
about a per-tile shift, the reference's epilogue and float64 per-image means; with ``data_range=None`` a pre-pass computes
the range on the device.  An update never synchronises the host.  Errors the host can see from shapes and arguments are
raised before any launch, with the reference's types and messages, in its order (DESIGN.md K20)."""
from __future__ import annotations

from collections.abc import Sequence
from typing import List, Optional, Union

import torch
from torch import Tensor
from torch.nn import functional as F  # noqa: N812
from typing_extensions import Literal

from metrics_b200 import _native
from metrics_b200.utilities.checks import _check_same_shape
from metrics_b200.utilities.distributed import reduce

_EMPTY_MAX = ("max(): Expected reduction dim to be specified for input.numel() == 0. Specify the reduction dim with the "
              "'dim' argument.")
_SCALAR_NAME = {torch.int64: "Long", torch.int32: "Int", torch.int16: "Short", torch.int8: "Char", torch.uint8: "Byte"}
_NO_GRAPH = ("metrics_b200: structural similarity runs in CUDA kernels that record no autograd graph "
             "(is_differentiable is False), and an input requires grad: compute it under torch.no_grad() or on detached "
             "inputs")


def _ssim_check_inputs(preds: Tensor, target: Tensor) -> tuple[Tensor, Tensor]:
    """Shape checks of the reference.  A floating-point ``target`` keeps its dtype: K20 rounds it to ``preds``' dtype
    on load.  Any other ``target`` is converted here, as the reference converts it."""
    if preds.dtype != target.dtype and not target.is_floating_point():
        target = target.to(preds.dtype)
    _check_same_shape(preds, target)
    if len(preds.shape) not in (4, 5):
        raise ValueError(
            "Expected `preds` and `target` to have BxCxHxW or BxCxDxHxW shape."
            f" Got preds: {preds.shape} and target: {target.shape}."
        )
    return preds, target


def _no_graph(preds: Tensor, target: Tensor, message: str = _NO_GRAPH) -> None:
    """The reference would build an autograd graph here; a kernel cannot, so say so instead of returning a constant."""
    if torch.is_grad_enabled() and (preds.requires_grad or target.requires_grad):
        raise RuntimeError(message)


def _filter_args(ndim: int, gaussian_kernel: bool, sigma, kernel_size, return_full_image: bool = False,
                 return_contrast_sensitivity: bool = False) -> tuple[list, list]:
    """Per-axis ``kernel_size`` and ``sigma`` lists, after the reference's argument checks in its order."""
    is_3d = ndim == 5
    if not isinstance(kernel_size, Sequence):
        kernel_size = 3 * [kernel_size] if is_3d else 2 * [kernel_size]
    if not isinstance(sigma, Sequence):
        sigma = 3 * [sigma] if is_3d else 2 * [sigma]
    for seq in (kernel_size, sigma):
        if len(seq) != ndim - 2:
            raise ValueError(
                f"`kernel_size` has dimension {len(kernel_size)}, but expected to be two less that target dimensionality,"
                f" which is: {ndim}"
            )
        if len(seq) not in (2, 3):
            raise ValueError(
                f"Expected `kernel_size` dimension to be 2 or 3. `kernel_size` dimensionality: {len(kernel_size)}"
            )
    if return_full_image and return_contrast_sensitivity:
        raise ValueError("Arguments `return_full_image` and `return_contrast_sensitivity` are mutually exclusive.")
    if any(x % 2 == 0 or x <= 0 for x in kernel_size):
        raise ValueError(f"Expected `kernel_size` to have odd positive number. Got {kernel_size}.")
    if any(y <= 0 for y in sigma):
        raise ValueError(f"Expected `sigma` to have positive number. Got {sigma}.")
    return list(kernel_size), list(sigma)


def _plan(shape, gaussian_kernel: bool, sigma: list, kernel_size: list) -> tuple[tuple, tuple, list]:
    """Per-axis (d, h, w) tap counts and reflect pads of K20, and the filter per axis as ``(kind, taps, sigma)``.

    2-D: the depth axis has one tap and no pad.  3-D: the gaussian's taps come from ``sigma`` on every axis, but the last
    axis is padded by ``(kernel_size[2] - 1) // 2``, as the reference pads it, so that axis's output size can differ from
    its input size."""
    gauss = [int(3.5 * s + 0.5) * 2 + 1 for s in sigma]
    sizes = gauss if gaussian_kernel else kernel_size
    pads = [(sizes[0] - 1) // 2, (sizes[1] - 1) // 2]
    if len(shape) == 5:
        pads.append((kernel_size[2] - 1) // 2)
        taps = list(sizes)
        axes = [("g", sizes[k], sigma[k]) if gaussian_kernel else ("u", sizes[k], None) for k in range(3)]
        return tuple(taps), tuple(pads), axes
    axes = [("u", 1, None)] + [("g", sizes[k], sigma[k]) if gaussian_kernel else ("u", sizes[k], None) for k in range(2)]
    return (1, sizes[0], sizes[1]), (0, pads[0], pads[1]), axes


_WEIGHTS: dict = {}  # filter taps and MS-SSIM betas on the device, made once


def _weights(axes: list, dtype: torch.dtype, device: torch.device) -> Tensor:
    """The separable filter in ``dtype`` on ``device``, one axis after the other: the reference's 1-D gaussian, computed
    with torch as it computes it, or ``1 / k``.  Cached per filter, dtype and device."""
    key = (tuple(axes), dtype, device)
    w = _WEIGHTS.get(key)
    if w is None:
        parts = []
        for kind, k, s in axes:
            if kind == "g":
                dist = torch.arange(start=(1 - k) / 2, end=(1 + k) / 2, step=1, dtype=dtype, device=device)
                g = torch.exp(-torch.pow(dist / s, 2) / 2)
                parts.append(g / g.sum())
            else:
                parts.append(torch.full((k,), 1.0 / k, dtype=dtype, device=device))
        w = _WEIGHTS[key] = torch.cat(parts)
    return w


def _raise_shape_errors(preds: Tensor, data_range, taps: tuple, pads: tuple) -> None:
    """The errors the reference meets from here on for this input's shape and dtype, raised by the same torch calls on
    zero-stride stand-ins of the shapes (nothing the size of the input is allocated, nothing is launched)."""
    dtype = preds.dtype
    if preds.shape[0] == 0 or preds.numel() == 0:
        if data_range is None:
            raise RuntimeError(_EMPTY_MAX)
    if not dtype.is_floating_point:
        if dtype == torch.bool and data_range is None:
            raise RuntimeError("Subtraction, the `-` operator, with two bool tensors is not supported. Use the `^` or "
                               "`logical_xor()` operator instead.")
        if dtype == torch.bool:
            raise NotImplementedError(f"\"reflection_pad{preds.ndim - 2}d\" not implemented for 'Bool'")
        raise RuntimeError(f"expected scalar type {_SCALAR_NAME.get(dtype, dtype)} but found Float")
    spatial = list(preds.shape[2:])
    is_3d = preds.ndim == 5
    in_pads = list(pads if is_3d else pads[1:])
    # the reflect pad rejects pads not below a size, and any empty dimension but the batch
    if preds.numel() == 0 or any(p >= n for p, n in zip(in_pads, spatial)):
        stand_in = torch.zeros((), dtype=torch.float32).expand(*preds.shape)
        F.pad(stand_in, tuple(p for p in reversed(in_pads) for _ in range(2)), mode="reflect")
    out = [n + 2 * p - k + 1 for n, p, k in zip(spatial, in_pads, taps if is_3d else taps[1:])]
    if any(o < 1 for o in out):
        padded = [n + 2 * p for n, p in zip(spatial, in_pads)]
        x = torch.zeros((), dtype=torch.float32).expand(1, preds.shape[1], *padded)
        k = torch.zeros((), dtype=torch.float32).expand(preds.shape[1], 1, *(taps if is_3d else taps[1:]))
        (F.conv3d if is_3d else F.conv2d)(x, k, groups=preds.shape[1])
    if preds.shape[0] == 0:
        raise IndexError("tuple index out of range")


def _ssim_update(
    preds: Tensor,
    target: Tensor,
    gaussian_kernel: bool = True,
    sigma: Union[float, Sequence[float]] = 1.5,
    kernel_size: Union[int, Sequence[int]] = 11,
    data_range: Optional[Union[float, tuple[float, float]]] = None,
    k1: float = 0.01,
    k2: float = 0.03,
    return_full_image: bool = False,
    return_contrast_sensitivity: bool = False,
) -> Union[Tensor, tuple[Tensor, Tensor]]:
    """Per-image SSIM in ``preds``' dtype, and the map or the per-image contrast term when asked: one K20 call."""
    kernel_size, sigma = _filter_args(preds.ndim, gaussian_kernel, sigma, kernel_size, return_full_image,
                                      return_contrast_sensitivity)
    sim, cs, img = _ssim_scale(preds, target, gaussian_kernel, sigma, kernel_size, data_range, k1, k2,
                               return_contrast_sensitivity, return_full_image)
    sim = sim.to(preds.dtype)
    if return_contrast_sensitivity:
        return sim, cs.to(preds.dtype)
    if return_full_image:
        return sim, img
    return sim


def _ssim_scale(preds: Tensor, target: Tensor, gaussian_kernel: bool, sigma: list, kernel_size: list, data_range,
                k1: float, k2: float, want_cs: bool, want_map: bool):
    """One K20 call on checked arguments: float64 per-image SSIM, contrast term (or None) and map (or None)."""
    taps, pads, axes = _plan(preds.shape, gaussian_kernel, sigma, kernel_size)
    _raise_shape_errors(preds, data_range, taps, pads)
    clamp = None
    if isinstance(data_range, tuple):
        clamp = (float(data_range[0]), float(data_range[1]))
        data_range = data_range[1] - data_range[0]
    weights = _weights(axes, preds.dtype, preds.device)
    sim, cs, img = _native.ssim(preds, target, weights, taps, pads, preds.ndim == 5, clamp,
                                None if data_range is None else float(data_range), k1, k2, want_cs, want_map)
    if img is not None and preds.ndim == 4:
        img = img.squeeze(2)
    return sim, cs, img


def _ssim_compute(
    similarities: Tensor,
    reduction: Literal["elementwise_mean", "sum", "none", None] = "elementwise_mean",
) -> Tensor:
    """Apply the specified reduction to pre-computed structural similarity."""
    return reduce(similarities, reduction)


def structural_similarity_index_measure(
    preds: Tensor,
    target: Tensor,
    gaussian_kernel: bool = True,
    sigma: Union[float, Sequence[float]] = 1.5,
    kernel_size: Union[int, Sequence[int]] = 11,
    reduction: Literal["elementwise_mean", "sum", "none", None] = "elementwise_mean",
    data_range: Optional[Union[float, tuple[float, float]]] = None,
    k1: float = 0.01,
    k2: float = 0.03,
    return_full_image: bool = False,
    return_contrast_sensitivity: bool = False,
) -> Union[Tensor, tuple[Tensor, Tensor]]:
    """Structural similarity of CUDA ``[B, C, H, W]`` or ``[B, C, D, H, W]`` float tensors (reference :210-292).

    Same arguments, results and errors as the reference.  Moments are taken about a local shift, so float32 inputs with
    a large level keep their accuracy; float16 / bfloat16 are computed in float32 and rounded once at the output.  Raises
    ``RuntimeError`` when grad mode is on and an input requires grad: the kernel records no graph."""
    preds, target = _ssim_check_inputs(preds, target)
    _no_graph(preds, target)
    similarity_pack = _ssim_update(preds, target, gaussian_kernel, sigma, kernel_size, data_range, k1, k2,
                                   return_full_image, return_contrast_sensitivity)
    if isinstance(similarity_pack, tuple):
        similarity, image = similarity_pack
        return _ssim_compute(similarity, reduction), image
    return _ssim_compute(similarity_pack, reduction)


def _multiscale_ssim_update(
    preds: Tensor,
    target: Tensor,
    gaussian_kernel: bool = True,
    sigma: Union[float, Sequence[float]] = 1.5,
    kernel_size: Union[int, Sequence[int]] = 11,
    data_range: Optional[Union[float, tuple[float, float]]] = None,
    k1: float = 0.01,
    k2: float = 0.03,
    betas: Union[tuple[float, float, float, float, float], tuple[float, ...]] = (
        0.0448,
        0.2856,
        0.3001,
        0.2363,
        0.1333,
    ),
    normalize: Optional[Literal["relu", "simple"]] = None,
) -> Tensor:
    """Per-image MS-SSIM: one K20 call per scale (the contrast term of scales 0 … n−2, SSIM at the last), one pool
    kernel between scales, and the reference's epilogue over the ``[n, B]`` values as torch ops."""
    is_3d = preds.ndim == 5
    if not isinstance(kernel_size, Sequence):
        kernel_size = 3 * [kernel_size] if is_3d else 2 * [kernel_size]
    if not isinstance(sigma, Sequence):
        sigma = 3 * [sigma] if is_3d else 2 * [sigma]
    if preds.size()[-1] < 2 ** len(betas) or preds.size()[-2] < 2 ** len(betas):
        raise ValueError(
            f"For a given number of `betas` parameters {len(betas)}, the image height and width dimensions must be"
            f" larger than or equal to {2 ** len(betas)}."
        )
    _betas_div = max(1, (len(betas) - 1)) ** 2
    if preds.size()[-2] // _betas_div <= kernel_size[0] - 1:
        raise ValueError(
            f"For a given number of `betas` parameters {len(betas)} and kernel size {kernel_size[0]},"
            f" the image height must be larger than {(kernel_size[0] - 1) * _betas_div}."
        )
    if preds.size()[-1] // _betas_div <= kernel_size[1] - 1:
        raise ValueError(
            f"For a given number of `betas` parameters {len(betas)} and kernel size {kernel_size[1]},"
            f" the image width must be larger than {(kernel_size[1] - 1) * _betas_div}."
        )
    kernel_size, sigma = _filter_args(preds.ndim, gaussian_kernel, sigma, kernel_size)
    # every scale's shape errors before the first launch, in the order the reference meets them
    shape = list(preds.shape)
    for _ in range(len(betas)):
        taps, pads, _axes = _plan(shape, gaussian_kernel, sigma, kernel_size)
        _raise_shape_errors(torch.zeros((), dtype=preds.dtype).expand(*shape), data_range, taps, pads)
        pooled = [n // 2 for n in shape[2:]]
        if any(n < 1 for n in pooled):
            (F.avg_pool3d if is_3d else F.avg_pool2d)(torch.zeros((), dtype=torch.float32).expand(*shape),
                                                      (2, 2, 2) if is_3d else (2, 2))
        shape = shape[:2] + pooled
    mcs_list: List[Tensor] = []
    x, y = preds, target
    for k in range(len(betas)):
        last = k == len(betas) - 1
        sim, cs, _ = _ssim_scale(x, y, gaussian_kernel, sigma, kernel_size, data_range, k1, k2, not last, False)
        mcs_list.append(sim if last else cs)
        if not last:
            x, y = _native.ssim_avg_pool(x, y, is_3d)
    mcs_stack = torch.stack(mcs_list)
    if normalize == "relu":
        mcs_stack = torch.relu(mcs_stack)
    if normalize == "simple":
        mcs_stack = (mcs_stack + 1) / 2
    # the reference's betas are a float32 tensor: their float32 values, applied in float64.  Cached per device: a copy
    # from host memory would synchronise every update
    key = ("betas", tuple(betas), mcs_stack.device)
    betas_t = _WEIGHTS.get(key)
    if betas_t is None:
        betas_t = _WEIGHTS[key] = torch.tensor(betas, dtype=torch.float32).double().view(-1, 1).to(mcs_stack.device)
    out_dtype = torch.promote_types(preds.dtype, torch.float32)
    return torch.prod(mcs_stack**betas_t, dim=0).to(out_dtype)


def _multiscale_ssim_compute(
    mcs_per_image: Tensor,
    reduction: Literal["elementwise_mean", "sum", "none", None] = "elementwise_mean",
) -> Tensor:
    """Apply the specified reduction to pre-computed multi-scale structural similarity."""
    return reduce(mcs_per_image, reduction)


def _check_msssim_args(betas, normalize) -> None:
    if not isinstance(betas, tuple):
        raise ValueError("Argument `betas` is expected to be of a type tuple.")
    if isinstance(betas, tuple) and not all(isinstance(beta, float) for beta in betas):
        raise ValueError("Argument `betas` is expected to be a tuple of floats.")
    if normalize and normalize not in ("relu", "simple"):
        raise ValueError("Argument `normalize` to be expected either `None` or one of 'relu' or 'simple'")


def multiscale_structural_similarity_index_measure(
    preds: Tensor,
    target: Tensor,
    gaussian_kernel: bool = True,
    sigma: Union[float, Sequence[float]] = 1.5,
    kernel_size: Union[int, Sequence[int]] = 11,
    reduction: Literal["elementwise_mean", "sum", "none", None] = "elementwise_mean",
    data_range: Optional[Union[float, tuple[float, float]]] = None,
    k1: float = 0.01,
    k2: float = 0.03,
    betas: tuple[float, ...] = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333),
    normalize: Optional[Literal["relu", "simple"]] = "relu",
) -> Tensor:
    """Multi-scale structural similarity of CUDA float tensors (reference :449-529).  Same arguments, results and
    errors as the reference; every scale runs on K20 and the epilogue over the ``[n, B]`` values is float64 torch ops,
    returned in ``promote_types(preds.dtype, float32)`` as the reference returns it."""
    _check_msssim_args(betas, normalize)
    preds, target = _ssim_check_inputs(preds, target)
    _no_graph(preds, target)
    mcs_per_image = _multiscale_ssim_update(preds, target, gaussian_kernel, sigma, kernel_size, data_range, k1, k2,
                                            betas, normalize)
    return _multiscale_ssim_compute(mcs_per_image, reduction)
