"""Inputs of the VIF and UQI goldens (tests/golden/vif_uqi.npz, made by tests/golden/make_golden_vif_uqi.py) and the
helpers the CPU tests share: the case table, the class / functional replay, and numpy stand-ins of `_native.vif_scale`,
`_native.vif_decimate` and `_native.uqi` built on the float64 oracles (oracle/vif.py, oracle/uqi.py)."""
from __future__ import annotations

import os

import numpy as np
import torch

from oracle import uqi as ouq
from oracle import vif as ovf

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "vif_uqi.npz")
DTYPES = {"f64": torch.float64, "f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}


def _flat_and_negative(rng, shape, level):
    """Flat blocks (the σ < eps branches) and a block where target is minus preds (g < 0)."""
    p = level * rng.random(shape)
    t = p + 0.1 * level * rng.standard_normal(shape)
    h, w = shape[-2] // 2, shape[-1] // 2
    p[..., :h, :w] = level * 0.5
    t[..., :h, :w] = level * 0.25
    t[..., h:, w:] = level - p[..., h:, w:] + 0.01 * level * rng.standard_normal(t[..., h:, w:].shape)
    return p, t


def offset_pair(level: float, noise: float, seed: int = 3, size: int = 64):
    """A smooth ramp at `level` plus gaussian noise, preds and target: float32 moments about zero cancel here."""
    rng = np.random.default_rng(seed)
    ramp = np.linspace(0, 1, size)
    base = level + ramp[:, None] + ramp[None, :]
    return ((base + noise * rng.standard_normal((size, size)))[None, None],
            (base + noise * rng.standard_normal((size, size)))[None, None])


def cases() -> list[dict]:
    """name, kind ("vif" / "uqi"), dtype key, two batches of float64 numpy inputs, keyword arguments."""
    rng = np.random.default_rng(2026)
    out = []

    def add(name, kind, batches, dtype="f64", **kw):
        out.append(dict(name=name, kind=kind, dtype=dtype, batches=batches, kwargs=kw))

    def noisy(shape, level=1.0, noise=0.1):
        p = level * rng.random(shape)
        return p, p + noise * level * rng.standard_normal(shape)

    add("vif_doc", "vif", [(rng.standard_normal((4, 3, 41, 41)), rng.standard_normal((4, 3, 41, 41))) for _ in range(2)])
    add("vif_41_c1", "vif", [noisy((2, 1, 41, 41), 255.0) for _ in range(2)])
    add("vif_odd", "vif", [noisy((2, 3, 47, 63), 255.0, 0.05) for _ in range(2)])
    add("vif_odd2", "vif", [noisy((1, 1, 53, 45), 1.0) for _ in range(2)])
    add("vif_flat_negative", "vif", [_flat_and_negative(rng, (2, 2, 48, 50), 255.0) for _ in range(2)])
    add("vif_sigma", "vif", [noisy((2, 1, 44, 44), 1.0) for _ in range(2)], sigma_n_sq=0.5)
    for key in ("f32", "f16", "bf16"):
        add(f"vif_{key}", "vif", [noisy((2, 2, 45, 47), 1.0) for _ in range(2)], dtype=key)
    add("uqi_doc", "uqi", [(lambda p: (p, 0.75 * p))(rng.random((4, 1, 16, 16))) for _ in range(2)])
    add("uqi_c3", "uqi", [noisy((2, 3, 24, 28)) for _ in range(2)])
    add("uqi_sum", "uqi", [noisy((2, 3, 24, 28)) for _ in range(2)], reduction="sum")
    add("uqi_none", "uqi", [noisy((2, 2, 20, 22)) for _ in range(2)], reduction="none")
    add("uqi_aniso", "uqi", [noisy((2, 1, 25, 31)) for _ in range(2)], kernel_size=(11, 5), sigma=(1.5, 0.8))
    add("uqi_aniso_none", "uqi", [noisy((2, 1, 25, 31)) for _ in range(2)], kernel_size=(3, 7), sigma=(0.7, 2.0),
        reduction="none")
    add("uqi_one_tap", "uqi", [noisy((2, 2, 16, 16)) for _ in range(2)], kernel_size=(1, 1), sigma=(1.0, 1.0))
    add("uqi_one_tap_sum", "uqi", [noisy((2, 2, 16, 16)) for _ in range(2)], kernel_size=(1, 3), sigma=(1.0, 1.0),
        reduction="sum")
    add("uqi_one_tap_none", "uqi", [noisy((2, 2, 16, 16)) for _ in range(2)], kernel_size=(3, 1), sigma=(1.0, 1.0),
        reduction="none")
    add("uqi_constant_target", "uqi", [(rng.random((2, 2, 20, 20)), np.full((2, 2, 20, 20), 0.5)) for _ in range(2)])
    add("uqi_flat_negative", "uqi", [_flat_and_negative(rng, (2, 1, 24, 24), 1.0) for _ in range(2)])
    for key in ("f32", "f16", "bf16"):
        add(f"uqi_{key}", "uqi", [noisy((2, 2, 24, 26)) for _ in range(2)], dtype=key)
    return out


def tensors(case: dict, device="cpu"):
    dtype = DTYPES[case["dtype"]]
    return [(torch.from_numpy(p).to(dtype).to(device), torch.from_numpy(t).to(dtype).to(device))
            for p, t in case["batches"]]


def load() -> dict:
    return dict(np.load(GOLDEN))


def run_case(case: dict, F_vif, S_vif, F_uqi, S_uqi, device="cpu") -> dict:  # noqa: N803
    """Functional on the first batch and the class over both batches: {key: numpy array}."""
    name, kw = case["name"], case["kwargs"]
    batches = tensors(case, device)
    out = {}
    if case["kind"] == "vif":
        r = F_vif.visual_information_fidelity(*batches[0], **kw)
        m = S_vif.VisualInformationFidelity(**kw).to(device)
    else:
        r = F_uqi.universal_image_quality_index(*batches[0], **kw)
        m = S_uqi.UniversalImageQualityIndex(**kw).to(device)
    out[f"{name}/functional"] = r.detach().float().cpu().numpy() if r.dtype == torch.bfloat16 else r.cpu().numpy()
    for p, t in batches:
        m.update(p, t)
    res = m.compute()
    out[f"{name}/compute"] = res.detach().float().cpu().numpy() if res.dtype == torch.bfloat16 else res.cpu().numpy()
    return out


def standin_vif_scale(preds, target, weights, taps, eps, sigma_n_sq):
    """`_native.vif_scale` on CPU tensors from the numpy oracle."""
    w = weights.double().numpy()[1:1 + taps[1]]
    w = w / w.sum()
    x, y = preds.double().numpy(), target.to(preds.dtype).double().numpy()
    _, _, vx, vy, cov = ovf._moments(x, y, w)
    a, b = ovf.scale_terms(vx, vy, cov, eps, sigma_n_sq)
    return torch.from_numpy(a.sum((-2, -1))), torch.from_numpy(b.sum((-2, -1)))


def standin_vif_decimate(preds, target, weights, taps):
    """`_native.vif_decimate` on CPU tensors."""
    w = weights.double().numpy()[:taps[0]]
    w = w / w.sum()
    return tuple(torch.from_numpy(ovf.decimate(v.double().numpy(), w)).to(preds.dtype) for v in (preds, target))


def standin_uqi(preds, target, weights, taps, pads, crop, eps, want_map):
    """`_native.uqi` on CPU tensors: per-image crop sums and the full map ``[b, c, 1, o_h, o_w]``."""
    w = weights.double().numpy()
    per_axis = [w[1:1 + taps[1]], w[1 + taps[1]:]]
    ks = (taps[1], taps[2])
    full, _ = ouq.uqi(preds.double().numpy(), target.double().numpy(), ks, (1.0, 1.0), eps, taps=per_axis,
                      unit_taps=True)
    cropped = full[..., crop[0]:full.shape[2] - crop[0], crop[1]:full.shape[3] - crop[1]]
    if crop[0] == 0 or crop[1] == 0:
        cropped = cropped[..., :0, :0]
    sums = torch.from_numpy(cropped.reshape(cropped.shape[0], -1).sum(1))
    return sums, torch.from_numpy(full[:, :, None]).to(preds.dtype) if want_map else None
