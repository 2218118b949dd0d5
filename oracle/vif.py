"""Oracles of pixel-domain visual information fidelity (reference: functional/image/vif.py).

`vif_per_channel` is a numpy float64 restatement: per scale the separable gaussian as a valid correlation, the
decimation ``[..., ::2, ::2]`` of scales 1-3, moments about each image's mean (exact in float64 where the reference's
float32 ``E[x²] − μ²`` cancels), the reference's masks in its order and the two log10 sums, per (image, channel).
`torch_chain_vif` is the reference's torch op chain on any device (dense 2-D filters, masks, sums), the yardstick on the
same GPU.  `filter_taps` gives each scale's 1-D taps computed in the input dtype as K21 receives them."""
from __future__ import annotations

import numpy as np
import torch
from torch.nn import functional as F  # noqa: N812

from oracle.ssim import _correlate

SCALES = tuple((2 ** (4 - s) + 1, (2.0 ** (4 - s) + 1) / 5) for s in range(4))


def filter_taps(dtype=torch.float64, device="cpu") -> list[np.ndarray]:
    """float64 values of each scale's 1-D gaussian ``exp(-x² / 2σ²)`` computed in `dtype` on `device` (unnormalised)."""
    out = []
    for n, sigma in SCALES:
        coords = torch.arange(float(n), dtype=dtype, device=device) - (n - 1) / 2
        out.append(torch.exp(-(coords**2) / (2.0 * sigma**2)).double().cpu().numpy())
    return out


def _filter2(x: np.ndarray, w: np.ndarray) -> np.ndarray:
    return _correlate(_correlate(x, w, x.ndim - 2), w, x.ndim - 1)


def _moments(x: np.ndarray, y: np.ndarray, w: np.ndarray):
    """Means, variances (unclamped) and covariance of the separable filter `w` ⊗ `w` of total weight S, about each
    image's mean: the terms in (1 − S) that the shift leaves out are added back, so nothing cancels."""
    s = float(np.sum(w)) ** 2
    miss = 1.0 - s
    mx_, my_ = (v.reshape(v.shape[0], v.shape[1], -1).mean(-1)[..., None, None] for v in (x, y))
    xs, ys = x - mx_, y - my_
    fx, fy, fxx, fyy, fxy = (_filter2(v, w) for v in (xs, ys, xs * xs, ys * ys, xs * ys))
    mux, muy = fx + s * mx_, fy + s * my_
    vx = (fxx - fx * fx) + miss * (2 * mx_ * fx + s * mx_ * mx_)
    vy = (fyy - fy * fy) + miss * (2 * my_ * fy + s * my_ * my_)
    cov = (fxy - fx * fy) + miss * (mx_ * fy + my_ * fx + s * mx_ * my_)
    return mux, muy, vx, vy, cov


def scale_terms(sp: np.ndarray, st: np.ndarray, cov: np.ndarray, eps: float, sigma_n_sq: float):
    """The reference's masks in its order on float64 preds variance `sp`, target variance `st` and covariance: the two
    log10 terms per position."""
    sp, st = np.maximum(sp, 0.0), np.maximum(st, 0.0)
    with np.errstate(all="ignore"):
        g = cov / (st + eps)
        sv = sp - g * cov
        m = st < eps
        g, sv, st = np.where(m, 0.0, g), np.where(m, sp, sv), np.where(m, 0.0, st)
        m = sp < eps
        g, sv = np.where(m, 0.0, g), np.where(m, 0.0, sv)
        m = g < 0
        sv, g = np.where(m, sp, sv), np.where(m, 0.0, g)
        sv = np.where(np.isnan(sv), sv, np.maximum(sv, eps))
        return np.log10(1.0 + g * g * st / (sv + sigma_n_sq)), np.log10(1.0 + st / sigma_n_sq)


def decimate(x: np.ndarray, w: np.ndarray) -> np.ndarray:
    """``conv2d(x, w ⊗ w)[..., ::2, ::2]``."""
    return _filter2(x, w)[..., ::2, ::2]


def vif_per_channel(preds: np.ndarray, target: np.ndarray, sigma_n_sq: float = 2.0, eps: float = 1e-10, taps=None,
                    unit_taps: bool = True, round_to=None) -> np.ndarray:
    """float64 ``[B, C]`` VIF-P of float64 ``[B, C, H, W]`` inputs that already carry their dtype's rounding.

    ``taps``: each scale's 1-D taps (default: computed in float64); ``unit_taps`` divides them by their sum, as K21 does
    and as the reference's 2-D filter is divided by its sum.  ``round_to``: a torch dtype each decimated scale is rounded
    to, as the reference's convolution output is.  ``eps`` and ``sigma_n_sq`` as the caller rounded them."""
    x, y = np.asarray(preds, np.float64), np.asarray(target, np.float64)
    taps = [np.asarray(w, np.float64) for w in (filter_taps() if taps is None else taps)]
    if unit_taps:
        taps = [w / np.sum(w) for w in taps]
    pv = np.zeros(x.shape[:2])
    tv = np.zeros(x.shape[:2])
    for s, w in enumerate(taps):
        if s > 0:
            x, y = decimate(x, w), decimate(y, w)
            if round_to is not None:
                x = torch.from_numpy(x).to(round_to).double().numpy()
                y = torch.from_numpy(y).to(round_to).double().numpy()
        _, _, vx, vy, cov = _moments(x, y, w)
        a, b = scale_terms(vx, vy, cov, eps, sigma_n_sq)
        pv += a.sum((-2, -1))
        tv += b.sum((-2, -1))
    with np.errstate(all="ignore"):
        return pv / tv


def torch_chain_vif(preds: torch.Tensor, target: torch.Tensor, sigma_n_sq: float = 2.0) -> torch.Tensor:
    """The reference's op chain on the inputs' device, ``[B, C]`` in the inputs' dtype: per channel and scale the dense
    2-D gaussian, the five convolutions, the masks and the sums."""
    dtype, dev = preds.dtype, preds.device
    eps = torch.tensor(1e-10, dtype=dtype, device=dev)
    sn = torch.tensor(sigma_n_sq, dtype=dtype, device=dev)
    out = []
    for ch in range(preds.size(1)):
        x, y = preds[:, ch:ch + 1], target[:, ch:ch + 1]
        num = torch.zeros(1, dtype=dtype, device=dev)
        den = torch.zeros(1, dtype=dtype, device=dev)
        for s, (n, sigma) in enumerate(SCALES):
            c = (torch.arange(float(n), dtype=dtype, device=dev) - (n - 1) / 2) ** 2
            k = torch.exp(-(c[None, :] + c[:, None]) / (2.0 * sigma**2))
            k = (k / k.sum())[None, None]
            if s > 0:
                y, x = F.conv2d(y, k)[:, :, ::2, ::2], F.conv2d(x, k)[:, :, ::2, ::2]
            mt, mp = F.conv2d(y, k), F.conv2d(x, k)
            st = torch.clamp(F.conv2d(y * y, k) - mt**2, min=0.0)
            sp = torch.clamp(F.conv2d(x * x, k) - mp**2, min=0.0)
            cov = F.conv2d(y * x, k) - mt * mp
            g = cov / (st + eps)
            sv = sp - g * cov
            m = st < eps
            g, sv, st = torch.where(m, 0, g), torch.where(m, sp, sv), torch.where(m, 0, st)
            m = sp < eps
            g, sv = torch.where(m, 0, g), torch.where(m, 0, sv)
            m = g < 0
            sv, g = torch.where(m, sp, sv), torch.where(m, 0, g)
            sv = torch.clamp(sv, min=eps)
            num = num + torch.log10(1.0 + g**2.0 * st / (sv + sn)).sum((1, 2, 3))
            den = den + torch.log10(1.0 + st / sn).sum((1, 2, 3))
        out.append(num / den)
    return torch.stack(out, 1)
