"""Pixel-domain visual information fidelity, VIF-P (reference: functional/image/vif.py).

Each of the four scales is one call of kernel K21 (`mb200_vif_scale_update`): K20's windowed moments of the scale's
separable gaussian, valid filtering, the reference's masks and the two log10 terms summed per (image, channel) in
float64.  Scales 1-3 first run `mb200_vif_decimate`, the reference's ``conv2d(x, k)[..., ::2, ::2]``.  An update never
synchronises the host.  Errors that follow from shapes and dtypes are raised before any launch by the same torch call on
a stand-in (DESIGN.md K21)."""
from __future__ import annotations

import torch
from torch import Tensor
from torch.nn import functional as F  # noqa: N812

from metrics_b200 import _native
from metrics_b200.functional.image.ssim import _no_graph
from metrics_b200.utilities.checks import _check_same_shape

_NO_GRAPH = ("metrics_b200: visual information fidelity runs in CUDA kernels that record no autograd graph "
             "(is_differentiable is False), and an input requires grad: compute it under torch.no_grad() or on detached "
             "inputs")
# (taps, sigma) of the reference's four scales: n = 2^(4 - scale) + 1, sigma = n / 5
SCALES = tuple((2 ** (4 - s) + 1, (2.0 ** (4 - s) + 1) / 5) for s in range(4))
_CACHE: dict = {}  # per (dtype, device): each scale's taps; per dtype: eps and sigma_n_sq rounded to it


def _filter(win_size: float, sigma: float, dtype: torch.dtype, device) -> Tensor:
    """The reference's 2-D gaussian, as it computes it (only run on small stand-ins, to raise its errors)."""
    coords = torch.arange(win_size, dtype=dtype, device=device) - (win_size - 1) / 2
    g = coords**2
    g = torch.exp(-(g.unsqueeze(0) + g.unsqueeze(1)) / (2.0 * sigma**2))
    g /= torch.sum(g)
    return g


def _scale_weights(dtype: torch.dtype, device: torch.device) -> list:
    """Per scale: the 1-D gaussian ``exp(-x² / 2σ²)`` in ``dtype`` as ``[1, g, g]`` (depth, h, w).  The reference's
    2-D filter is their outer product divided by its sum; K21 divides each axis by its sum, so the products agree."""
    key = (dtype, device)
    ws = _CACHE.get(key)
    if ws is None:
        ws = []
        for n, sigma in SCALES:
            coords = torch.arange(float(n), dtype=dtype, device=device) - (n - 1) / 2
            g = torch.exp(-(coords**2) / (2.0 * sigma**2))
            ws.append(torch.cat([torch.ones(1, dtype=dtype, device=device), g, g]))
        ws = _CACHE[key] = ws
    return ws


def _constants(dtype: torch.dtype, sigma_n_sq: float) -> tuple[float, float]:
    """``eps = 1e-10`` and ``sigma_n_sq`` rounded to ``dtype`` as ``torch.tensor(..., dtype=dtype)`` rounds them
    (float16: eps is 0).  Host tensors only: nothing touches the device."""
    key = ("consts", dtype, float(sigma_n_sq))
    c = _CACHE.get(key)
    if c is None:
        c = _CACHE[key] = (torch.tensor(1e-10, dtype=dtype).item(), torch.tensor(sigma_n_sq, dtype=dtype).item())
    return c


def _conv(h: int, w: int, n: int) -> None:
    """A valid ``n x n`` convolution of an ``h x w`` image: conv2d's error when the image is smaller, from a stand-in."""
    if h < n or w < n:
        F.conv2d(torch.zeros((), dtype=torch.float32).expand(1, 1, h, w),
                 torch.zeros((), dtype=torch.float32).expand(1, 1, n, n))


def _raise_vif_errors(preds: Tensor, target: Tensor) -> None:
    """The errors the reference's channel loop meets for these shapes and dtypes, in its order, raised by the same torch
    calls on zero-stride stand-ins (nothing the size of the input is allocated, nothing is launched)."""
    if preds.ndim < 4:
        torch.zeros((), dtype=torch.float32).expand(*preds.shape)[:, 0, :, :]  # IndexError: too many indices
    if preds.size(1) == 0:
        torch.cat([])
    if not preds.dtype.is_floating_point or target.dtype != preds.dtype or preds.ndim != 4:
        # the first scale's filter and its convolutions of target, then preds: each of these raises here
        kernel = _filter(17.0, 17 / 5, dtype=preds.dtype, device="cpu")[None, None, :]
        F.conv2d(torch.zeros((), dtype=target.dtype).expand(target.shape[0], 1, *target.shape[2:]), kernel)
        F.conv2d(torch.zeros((), dtype=preds.dtype).expand(preds.shape[0], 1, *preds.shape[2:]), kernel)
        raise TypeError(f"metrics_b200: visual information fidelity needs 4-D float inputs of one dtype, got "
                        f"{preds.dtype} {tuple(preds.shape)} and {target.dtype} {tuple(target.shape)}")
    # K21 reads both inputs through one geometry; the reference would filter inputs of different shapes separately
    _check_same_shape(preds, target)
    h, w = preds.shape[2:]
    for s, (n, _) in enumerate(SCALES):
        if s > 0:
            _conv(h, w, n)  # the decimation
            h, w = (h - n + 2) // 2, (w - n + 2) // 2
        _conv(h, w, n)  # the moments


def _vif_per_channel(preds: Tensor, target: Tensor, sigma_n_sq: float) -> Tensor:
    """``[B, C]`` VIF-P per image and channel in ``preds``' dtype: the float64 sums of each term over the four scales,
    added in scale order, and their ratio, rounded once."""
    _raise_vif_errors(preds, target)
    dtype = preds.dtype
    eps, sn = _constants(dtype, sigma_n_sq)
    ws = _scale_weights(dtype, preds.device)
    x, y = preds, target
    sums = []
    for s, (n, _) in enumerate(SCALES):
        if s > 0:
            x, y = _native.vif_decimate(x, y, ws[s][1:], (n, n))
        sums.append(torch.stack(_native.vif_scale(x, y, ws[s], (1, n, n), eps, sn)))
    total = torch.stack(sums).sum(0)  # [2, B, C]: the scales in order, per element
    return (total[0] / total[1]).to(dtype)


def visual_information_fidelity(preds: Tensor, target: Tensor, sigma_n_sq: float = 2.0) -> Tensor:
    """Pixel-based visual information fidelity of CUDA ``[N, C, H, W]`` float tensors, ``H, W >= 41`` (reference
    :86-115): the mean over every (image, channel) of its VIF-P, in the inputs' dtype.

    Variances are taken about a per-tile shift (K20), so the masks that compare them with ``eps`` are decided on accurate
    values; float16 / bfloat16 are computed in float32.  Raises ``RuntimeError`` when grad mode is on and an input
    requires grad: the kernels record no graph."""
    if preds.size(-1) < 41 or preds.size(-2) < 41:
        raise ValueError(f"Invalid size of preds. Expected at least 41x41, but got {preds.size(-1)}x{preds.size(-2)}!")
    if target.size(-1) < 41 or target.size(-2) < 41:
        raise ValueError(
            f"Invalid size of target. Expected at least 41x41, but got {target.size(-1)}x{target.size(-2)}!"
        )
    _no_graph(preds, target, _NO_GRAPH)
    return _vif_per_channel(preds, target, sigma_n_sq).mean()
