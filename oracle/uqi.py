"""Oracles of the universal image quality index (reference: functional/image/uqi.py).

`uqi` is a numpy float64 restatement: reflect padding (the width by ``pad_h``, the height by ``pad_w``, as the reference
pads), the separable gaussian as a valid correlation, moments about each image's mean, the map and the reference's crop
``[pad_h : −pad_h, pad_w : −pad_w]``.  `torch_chain_uqi` is the reference's torch op chain (pad, five-image cat, grouped
conv, epilogue, crop) on any device, the yardstick on the same GPU."""
from __future__ import annotations

import numpy as np
import torch
from torch.nn import functional as F  # noqa: N812

from oracle.ssim import _correlate, filter_taps


def axes(kernel_size=(11, 11), sigma=(1.5, 1.5)) -> list:
    return [("g", kernel_size[0], sigma[0]), ("g", kernel_size[1], sigma[1])]


def uqi(preds: np.ndarray, target: np.ndarray, kernel_size=(11, 11), sigma=(1.5, 1.5), eps: float = None, taps=None,
        unit_taps: bool = False):
    """float64 (full map, cropped map) of float64 ``[B, C, H, W]`` inputs that already carry their dtype's rounding.
    ``eps``: the dtype's machine epsilon (default float32's, the reference's for float32 inputs).  ``taps``: per-axis
    taps (default: computed in float64), carried exactly with their total weight S; ``unit_taps`` divides them by
    their sum first, as K21 does."""
    p, t = np.asarray(preds, np.float64), np.asarray(target, np.float64)
    eps = float(torch.finfo(torch.float32).eps) if eps is None else eps
    taps = [np.asarray(w, np.float64) for w in (filter_taps(axes(kernel_size, sigma)) if taps is None else taps)]
    if unit_taps:
        taps = [w / np.sum(w) for w in taps]
    s = float(np.prod([np.sum(w) for w in taps]))
    miss = 1.0 - s
    pad_h, pad_w = (kernel_size[0] - 1) // 2, (kernel_size[1] - 1) // 2
    width = [(0, 0), (0, 0), (pad_w, pad_w), (pad_h, pad_h)]
    mp = p.reshape(p.shape[0], -1).mean(1).reshape(-1, 1, 1, 1) if p.size else np.zeros((p.shape[0], 1, 1, 1))
    mt = t.reshape(t.shape[0], -1).mean(1).reshape(-1, 1, 1, 1) if t.size else np.zeros((t.shape[0], 1, 1, 1))
    x, y = np.pad(p - mp, width, mode="reflect"), np.pad(t - mt, width, mode="reflect")

    def filt(img):
        return _correlate(_correlate(img, taps[0], 2), taps[1], 3)

    with np.errstate(all="ignore"):
        fx, fy, fxx, fyy, fxy = (filt(v) for v in (x, y, x * x, y * y, x * y))
        mux, muy = fx + s * mp, fy + s * mt
        vx = np.maximum((fxx - fx * fx) + miss * (2 * mp * fx + s * mp * mp), 0.0)
        vy = np.maximum((fyy - fy * fy) + miss * (2 * mt * fy + s * mt * mt), 0.0)
        cov = (fxy - fx * fy) + miss * (mp * fy + mt * fx + s * mp * mt)
        full = ((2 * mux * muy) * (2 * cov)) / ((mux * mux + muy * muy) * (vx + vy) + eps)
    return full, full[..., pad_h:-pad_h, pad_w:-pad_w]


def reduce(crop: np.ndarray, reduction):
    if reduction == "elementwise_mean":
        return np.mean(crop) if crop.size else np.float64(np.nan)
    if reduction == "sum":
        return np.sum(crop)
    return crop


def torch_chain_uqi(preds: torch.Tensor, target: torch.Tensor, kernel_size=(11, 11), sigma=(1.5, 1.5)) -> torch.Tensor:
    """The reference's op chain on the inputs' device: the cropped map in the inputs' dtype."""
    dtype, dev, ch = preds.dtype, preds.device, preds.size(1)
    parts = []
    for k, s in zip(kernel_size, sigma):
        dist = torch.arange(start=(1 - k) / 2, end=(1 + k) / 2, step=1, dtype=dtype, device=dev)
        g = torch.exp(-torch.pow(dist / s, 2) / 2)
        parts.append((g / g.sum())[None])
    kern = torch.matmul(parts[0].t(), parts[1]).expand(ch, 1, kernel_size[0], kernel_size[1])
    pad_h, pad_w = (kernel_size[0] - 1) // 2, (kernel_size[1] - 1) // 2
    p = F.pad(preds, (pad_h, pad_h, pad_w, pad_w), mode="reflect")
    t = F.pad(target, (pad_h, pad_h, pad_w, pad_w), mode="reflect")
    out = F.conv2d(torch.cat((p, t, p * p, t * t, p * t)), kern, groups=ch).split(p.shape[0])
    mpp, mtt, mpt = out[0].pow(2), out[1].pow(2), out[0] * out[1]
    sp = torch.clamp(out[2] - mpp, min=0.0)
    st = torch.clamp(out[3] - mtt, min=0.0)
    spt = out[4] - mpt
    eps = torch.finfo(sp.dtype).eps
    full = ((2 * mpt) * (2 * spt)) / ((mpp + mtt) * (sp + st) + eps)
    return full[..., pad_h:-pad_h, pad_w:-pad_w]
