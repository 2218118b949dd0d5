"""Oracles of structural similarity (reference: functional/image/ssim.py).

`ssim` is a numpy float64 restatement: reflect padding per axis, the separable filter as a valid correlation, moments
about each image's mean (exact in float64 where the reference's float32 cancels), the reference's epilogue, crops and
means.  `ms_ssim` chains it over the scales with the reference's average pool.  `torch_chain_ssim` is the reference's
torch op chain (pad, five-image cat, grouped conv, epilogue) on any device, the yardstick K20 is compared with on the
same GPU.  `filter_taps` gives the taps each axis uses, computed in the input dtype as the reference computes them."""
from __future__ import annotations

import warnings

import numpy as np
import torch
from torch.nn import functional as F  # noqa: N812


def plan(ndim: int, gaussian_kernel: bool, sigma, kernel_size):
    """Per spatial axis: (kind, taps, sigma) and reflect pad, as the reference derives them (3-D: the last axis is padded
    by (kernel_size[2] - 1) // 2 whatever its gaussian's size)."""
    n = ndim - 2
    ks = list(kernel_size) if isinstance(kernel_size, (list, tuple)) else [kernel_size] * n
    sg = list(sigma) if isinstance(sigma, (list, tuple)) else [sigma] * n
    gauss = [int(3.5 * s + 0.5) * 2 + 1 for s in sg]
    sizes = gauss if gaussian_kernel else ks
    pads = [(sizes[0] - 1) // 2, (sizes[1] - 1) // 2] + ([(ks[2] - 1) // 2] if n == 3 else [])
    axes = [("g", sizes[k], sg[k]) if gaussian_kernel else ("u", sizes[k], None) for k in range(n)]
    return axes, pads


def filter_taps(axes, dtype=torch.float64, device="cpu") -> list[np.ndarray]:
    """float64 values of each axis's taps as computed in `dtype` on `device` (the reference's 1-D gaussian, or 1 / k).
    In float16 / bfloat16 a tap can round differently on CPU and CUDA, so a GPU comparison takes them from the GPU."""
    out = []
    for kind, k, s in axes:
        if kind == "g":
            dist = torch.arange(start=(1 - k) / 2, end=(1 + k) / 2, step=1, dtype=dtype, device=device)
            g = torch.exp(-torch.pow(dist / s, 2) / 2)
            out.append((g / g.sum()).double().cpu().numpy())
        else:
            out.append(torch.full((k,), 1.0 / k, dtype=dtype).double().numpy())
    return out


def _correlate(x: np.ndarray, taps: np.ndarray, axis: int) -> np.ndarray:
    k = len(taps)
    n = x.shape[axis] - k + 1
    out = np.zeros(x.shape[:axis] + (n,) + x.shape[axis + 1:])
    for t in range(k):
        out += taps[t] * np.take(x, np.arange(t, t + n), axis=axis)
    return out


def ssim(preds: np.ndarray, target: np.ndarray, gaussian_kernel: bool = True, sigma=1.5, kernel_size=11,
         data_range=None, k1: float = 0.01, k2: float = 0.03, taps=None, pads=None, unit_taps: bool = False):
    """float64 (per-image SSIM [B], per-image contrast term over the crop [B], map) of float64 inputs that already carry
    their dtype's rounding.  ``taps``: per-axis filter taps (default: computed in float64); ``pads``: per-axis reflect
    pads (default: the reference's).

    The default is the reference's arithmetic carried out exactly with the taps as given, whose total weight S may miss 1
    (a float16 / bfloat16 gaussian by up to 1e-3, float32 taps by about 1e-7): the moments are taken about each image's
    mean and the terms in (1 − S) that a shift leaves out are added back, so no variance is formed as a difference of
    large numbers.  ``unit_taps`` divides each axis's taps by their sum first, as K20 does (S = 1)."""
    p, t = np.asarray(preds, np.float64), np.asarray(target, np.float64)
    axes, ref_pads = plan(p.ndim, gaussian_kernel, sigma, kernel_size)
    taps = [np.asarray(w, np.float64) for w in (filter_taps(axes) if taps is None else taps)]
    if unit_taps:
        taps = [w / np.sum(w) for w in taps]
    weight = float(np.prod([np.sum(w) for w in taps]))
    pads = ref_pads if pads is None else list(pads)
    if data_range is None:
        dr_p, dr_t = p.max() - p.min(), t.max() - t.min()
        data_range = dr_t if dr_t > dr_p else dr_p
    elif isinstance(data_range, tuple):
        p, t = np.clip(p, *data_range), np.clip(t, *data_range)
        data_range = data_range[1] - data_range[0]
    c1, c2 = (k1 * data_range) ** 2, (k2 * data_range) ** 2
    width = [(0, 0), (0, 0)] + [(q, q) for q in pads]
    shape = (p.shape[0],) + (1,) * (p.ndim - 1)

    def finite_mean(x):
        x = np.where(np.isfinite(x), x, np.nan).reshape(x.shape[0], -1)
        with np.errstate(all="ignore"), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            return np.nan_to_num(np.nanmean(x, 1), nan=0.0).reshape(shape)

    sp, st = finite_mean(p), finite_mean(t)
    with np.errstate(all="ignore"):
        x, y = np.pad(p - sp, width, mode="reflect"), np.pad(t - st, width, mode="reflect")
        moments = []
        for img in (x, y, x * x, y * y, x * y):
            for a, w in enumerate(taps):
                img = _correlate(img, w, a + 2)
            moments.append(img)
        mx, my, mxx, myy, mxy = moments
        miss = 1.0 - weight
        mux, muy = mx + weight * sp, my + weight * st
        vx_raw = (mxx - mx * mx) + miss * (2 * sp * mx + weight * sp * sp)
        vy_raw = (myy - my * my) + miss * (2 * st * my + weight * st * st)
        cov = (mxy - mx * my) + miss * (sp * my + st * mx + weight * sp * st)
        vx = np.where(np.isnan(vx_raw), np.nan, np.maximum(vx_raw, 0.0))
        vy = np.where(np.isnan(vy_raw), np.nan, np.maximum(vy_raw, 0.0))
        upper = 2 * cov + c2
        lower = (vx + vy) + c2
        full = ((2 * mux * muy + c1) * upper) / ((mux * mux + muy * muy + c1) * lower)
        crop = (slice(None), slice(None)) + tuple(slice(q, -q) for q in pads)
        cs = (upper / lower)[crop]
        b = p.shape[0]
        sim = full.reshape(b, -1).mean(1)
        csm = cs.reshape(b, -1).mean(1) if cs.size else np.full(b, np.nan)
    return sim, csm, full


def avg_pool(x: np.ndarray) -> np.ndarray:
    """2x2 (4-D) or 2x2x2 (5-D) average pool with floor sizes."""
    for a in range(2, x.ndim):
        n = x.shape[a] // 2
        x = 0.5 * (np.take(x, np.arange(0, 2 * n, 2), axis=a) + np.take(x, np.arange(1, 2 * n, 2), axis=a))
    return x


def ms_ssim(preds, target, gaussian_kernel=True, sigma=1.5, kernel_size=11, data_range=None, k1=0.01, k2=0.03,
            betas=(0.0448, 0.2856, 0.3001, 0.2363, 0.1333), normalize="relu", taps=None, round_to=None,
            unit_taps: bool = False):
    """float64 per-image MS-SSIM.  ``round_to``: a torch dtype each pooled scale is rounded to, as the reference pools in
    the input dtype; ``taps`` / ``unit_taps`` as for `ssim`."""
    p, t = np.asarray(preds, np.float64), np.asarray(target, np.float64)
    vals = []
    for k in range(len(betas)):
        sim, cs, _ = ssim(p, t, gaussian_kernel, sigma, kernel_size, data_range, k1, k2, taps, unit_taps=unit_taps)
        vals.append(sim if k == len(betas) - 1 else cs)
        p, t = avg_pool(p), avg_pool(t)
        if round_to is not None:
            p = torch.from_numpy(p).to(round_to).double().numpy()
            t = torch.from_numpy(t).to(round_to).double().numpy()
    stack = np.stack(vals)
    if normalize == "relu":
        stack = np.maximum(stack, 0.0)
    if normalize == "simple":
        stack = (stack + 1) / 2
    with np.errstate(invalid="ignore"):
        # the reference's betas are a float32 tensor
        return np.prod(stack ** np.asarray(betas, np.float32).astype(np.float64).reshape(-1, 1), axis=0)


def torch_chain_ssim(preds: torch.Tensor, target: torch.Tensor, gaussian_kernel: bool = True, sigma=1.5,
                     kernel_size=11, data_range=None, k1: float = 0.01, k2: float = 0.03):
    """The reference's op chain on the inputs' device: (per-image SSIM, per-image contrast term, map) in the inputs'
    dtype.  With data_range=None it synchronises the host, as the reference does."""
    target = target.to(preds.dtype)
    is_3d = preds.ndim == 5
    axes, pads = plan(preds.ndim, gaussian_kernel, sigma, kernel_size)
    if data_range is None:
        data_range = max(preds.max() - preds.min(), target.max() - target.min())
    elif isinstance(data_range, tuple):
        preds = torch.clamp(preds, min=data_range[0], max=data_range[1])
        target = torch.clamp(target, min=data_range[0], max=data_range[1])
        data_range = data_range[1] - data_range[0]
    c1, c2 = pow(k1 * data_range, 2), pow(k2 * data_range, 2)
    dtype, dev, ch = preds.dtype, preds.device, preds.size(1)
    fpad = tuple(q for q in reversed(pads) for _ in range(2))
    preds, target = F.pad(preds, fpad, mode="reflect"), F.pad(target, fpad, mode="reflect")
    if gaussian_kernel:
        kern = None
        for kind, k, s in axes:
            dist = torch.arange(start=(1 - k) / 2, end=(1 + k) / 2, step=1, dtype=dtype, device=dev)
            g = torch.exp(-torch.pow(dist / s, 2) / 2)
            g = g / g.sum()
            kern = g if kern is None else kern.unsqueeze(-1) * g
    else:
        sizes = [k for _, k, _ in axes]
        kern = torch.ones(sizes, dtype=dtype, device=dev) / torch.prod(torch.tensor(sizes, dtype=dtype, device=dev))
    kern = kern.expand(ch, 1, *kern.shape)
    both = torch.cat((preds, target, preds * preds, target * target, preds * target))
    out = (F.conv3d if is_3d else F.conv2d)(both, kern, groups=ch).split(preds.shape[0])
    mu_p2, mu_t2, mu_pt = out[0].pow(2), out[1].pow(2), out[0] * out[1]
    s_p = torch.clamp(out[2] - mu_p2, min=0.0)
    s_t = torch.clamp(out[3] - mu_t2, min=0.0)
    s_pt = out[4] - mu_pt
    upper = 2 * s_pt.to(dtype) + c2
    lower = (s_p + s_t).to(dtype) + c2
    full = ((2 * mu_pt + c1) * upper) / ((mu_p2 + mu_t2 + c1) * lower)
    cs = upper / lower
    cs = cs[(Ellipsis,) + tuple(slice(q, -q) for q in pads)]
    b = full.shape[0]
    return full.reshape(b, -1).mean(-1), cs.reshape(cs.shape[0], -1).mean(-1), full
