"""Inputs of the structural-similarity goldens (tests/golden/ssim.npz, made by tests/golden/make_golden_ssim.py) and the
helpers the CPU tests share: the case table, the class / functional replay, and numpy stand-ins of `_native.ssim` and
`_native.ssim_avg_pool` built on the float64 oracle (oracle/ssim.py)."""
from __future__ import annotations

import os

import numpy as np
import torch

from oracle import ssim as osm

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "ssim.npz")
MS_BETAS3 = (0.2, 0.3, 0.5)


def _pair(rng: np.random.Generator, shape, level: float = 0.0, noise: float = 0.1):
    p = rng.random(shape) + level
    return p, p + noise * rng.standard_normal(shape)


def offset_pair(level: float, noise: float, seed: int = 3):
    """A smooth 128 x 128 ramp at `level` plus gaussian noise of `noise`, preds and target: float32 SSIM about zero
    cancels here."""
    rng = np.random.default_rng(seed)
    ramp = np.linspace(0, 1, 128)
    base = level + ramp[:, None] + ramp[None, :]
    return ((base + noise * rng.standard_normal((128, 128)))[None, None],
            (base + noise * rng.standard_normal((128, 128)))[None, None])


def cases() -> list[dict]:
    """name, kind ("ssim" / "ms"), two batches of float64 numpy inputs, keyword arguments of the reference call."""
    rng = np.random.default_rng(2025)
    out = []

    def add(name, shape, kind="ssim", **kw):
        out.append(dict(name=name, kind=kind, batches=[_pair(rng, shape), _pair(rng, shape)], kwargs=kw))

    add("gauss", (2, 3, 24, 28))
    add("gauss_range1", (2, 3, 24, 28), data_range=1.0)
    add("tuple_clamp", (2, 2, 20, 22), data_range=(0.2, 0.7))
    add("uniform", (2, 2, 20, 22), gaussian_kernel=False, kernel_size=(3, 7))
    add("anisotropic", (2, 1, 25, 31), sigma=(0.7, 2.0))
    add("one_tap_axis", (2, 1, 16, 16), gaussian_kernel=False, kernel_size=(1, 5), return_contrast_sensitivity=True)
    add("contrast", (2, 3, 24, 28), return_contrast_sensitivity=True)
    add("full_image", (2, 3, 24, 28), data_range=1.0, return_full_image=True)
    add("sum", (2, 3, 24, 28), reduction="sum")
    add("none", (2, 3, 24, 28), reduction="none", data_range=1.0)
    add("3d", (1, 2, 9, 10, 12), kernel_size=(3, 3, 5), sigma=(0.5, 0.5, 0.5), data_range=1.0)
    add("3d_gauss_ne_ks", (1, 1, 9, 14, 16), kernel_size=(3, 3, 3), sigma=(0.6, 0.8, 1.5), return_full_image=True)
    add("ms", (2, 1, 180, 180), kind="ms", data_range=1.0)
    add("ms_betas3_simple", (2, 2, 48, 52), kind="ms", betas=MS_BETAS3, normalize="simple", kernel_size=5, sigma=0.8)
    add("ms_none_normalize", (1, 1, 48, 52), kind="ms", betas=MS_BETAS3, normalize=None, kernel_size=5, sigma=0.8,
        data_range=1.0)
    add("ms_3d", (1, 1, 8, 32, 32), kind="ms", betas=(0.5, 0.5), kernel_size=3, sigma=0.5, data_range=1.0)
    return out


def tensors(case: dict, dtype=torch.float64, device="cpu"):
    return [(torch.from_numpy(p).to(dtype).to(device), torch.from_numpy(t).to(dtype).to(device))
            for p, t in case["batches"]]


def load() -> dict:
    return dict(np.load(GOLDEN))


def run_case(case: dict, F, S, dtype=torch.float64, device="cpu") -> dict:  # noqa: N803
    """Functional on the first batch and the class over both batches: {key: numpy array}."""
    name, kw = case["name"], case["kwargs"]
    batches = tensors(case, dtype, device)
    out = {}
    if case["kind"] == "ssim":
        r = F.structural_similarity_index_measure(*batches[0], **kw)
        m = S.StructuralSimilarityIndexMeasure(**kw)
    else:
        r = F.multiscale_structural_similarity_index_measure(*batches[0], **kw)
        m = S.MultiScaleStructuralSimilarityIndexMeasure(**kw)
    if isinstance(r, tuple):
        out[f"{name}/functional"], out[f"{name}/functional_image"] = (x.detach().cpu().numpy() for x in r)
    else:
        out[f"{name}/functional"] = r.detach().cpu().numpy()
    m = m.to(device)
    for p, t in batches:
        m.update(p, t)
    res = m.compute()
    if isinstance(res, tuple):
        out[f"{name}/compute"], out[f"{name}/compute_image"] = (x.detach().cpu().numpy() for x in res)
    else:
        out[f"{name}/compute"] = res.detach().cpu().numpy()
    out[f"{name}/total"] = m.total.detach().cpu().numpy()
    return out


def standin_ssim(preds, target, weights, taps, pads, crop_depth, clamp, data_range, k1, k2, want_cs, want_map):
    """`_native.ssim` on CPU tensors from the numpy oracle: same outputs, same shapes and dtypes."""
    w = weights.double().numpy()
    cuts = np.cumsum(taps)[:-1]
    per_axis = np.split(w, cuts)
    if preds.ndim == 4:
        per_axis = per_axis[1:]
    p = preds.double().numpy()
    t = target.to(preds.dtype).double().numpy()
    dr = clamp if clamp is not None else data_range
    in_pads = list(pads[1:]) if preds.ndim == 4 else list(pads)
    sim, cs, full = osm.ssim(p, t, data_range=dr, k1=k1, k2=k2, taps=per_axis, pads=in_pads, unit_taps=True)
    if preds.ndim == 4:
        full = full[:, :, None]
    return (torch.from_numpy(sim), torch.from_numpy(cs) if want_cs else None,
            torch.from_numpy(full).to(preds.dtype) if want_map else None)


def standin_pool(preds, target, pool_depth):
    """`_native.ssim_avg_pool` on CPU tensors."""
    def pool(x):
        x = x.to(preds.dtype).double()
        if x.ndim == 5 and not pool_depth:
            return torch.nn.functional.avg_pool3d(x, (1, 2, 2)).to(preds.dtype)
        return (torch.nn.functional.avg_pool3d(x, 2) if x.ndim == 5 else torch.nn.functional.avg_pool2d(x, 2)).to(preds.dtype)

    return pool(preds), pool(target)
