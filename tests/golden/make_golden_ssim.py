"""Generate tests/golden/ssim.npz and tests/golden/ssim_surface.json from the UNMODIFIED reference (TorchMetrics under
/root/reference), CPU tensors.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_ssim.py

Same import set-up as make_golden.py.  Every case of tests/ssim_cases.py goes through the reference functional on its
first batch and the reference class over both batches, in float64.  The offset workloads (a ramp at level 0, 100 and 1000
plus noise) are recorded in float64 and in the reference's float32, which is wrong there.  The json holds the signatures,
the class attributes, the state registry and the reference's error types and messages.
"""
from __future__ import annotations

import importlib
import inspect
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
ATTRS = ("is_differentiable", "higher_is_better", "full_state_update", "plot_lower_bound", "plot_upper_bound")
CLASSES = ("StructuralSimilarityIndexMeasure", "MultiScaleStructuralSimilarityIndexMeasure")
FUNCTIONALS = ("structural_similarity_index_measure", "multiscale_structural_similarity_index_measure")
OFFSETS = ((0.0, 1e-3), (100.0, 1e-3), (1000.0, 1e-2))


def _signature(fn):
    sig = inspect.signature(fn)
    return [[n, "<required>" if p.default is inspect.Parameter.empty else repr(p.default)] for n, p in sig.parameters.items()
            if n != "self"]


def ssim_surface(pkg: str) -> dict:
    S = importlib.import_module(f"{pkg}.image.ssim")  # noqa: N806
    F = importlib.import_module(f"{pkg}.functional.image.ssim")  # noqa: N806
    out = {}
    for name in CLASSES:
        cls = getattr(S, name)
        out[f"image.{name}"] = {"init": _signature(cls.__init__), "update": _signature(cls.update),
                                "compute": _signature(cls.compute), "attrs": {a: repr(getattr(cls, a, None)) for a in ATTRS}}
    for name in FUNCTIONALS:
        out[f"functional.image.{name}"] = {"call": _signature(getattr(F, name))}
    return out


def ssim_states(pkg: str) -> dict:
    S = importlib.import_module(f"{pkg}.image.ssim")  # noqa: N806
    out = {}
    for name in CLASSES:
        for label, kw in (("mean", {}), ("none", {"reduction": "none"}), ("image", {"return_full_image": True})):
            if name.startswith("Multi") and label == "image":
                continue
            m = getattr(S, name)(**kw)
            out[f"{name}/{label}"] = {
                k: {"default": [list(v.shape), str(v.dtype)] if isinstance(v, torch.Tensor) else repr(v),
                    "reduce": getattr(m._reductions[k], "__name__", None), "persistent": m._persistent[k]}
                for k, v in m._defaults.items()}
    return out


def error_calls(F, S):  # noqa: N803
    """name -> call, for the functional module F and the class module S of either package (CPU inputs: every one of
    these errors is raised before any data is read)."""
    x = torch.rand(2, 3, 16, 16)
    v = torch.rand(1, 1, 8, 9, 12)
    big = torch.rand(1, 1, 64, 64)
    fs, fm = F.structural_similarity_index_measure, F.multiscale_structural_similarity_index_measure
    return {
        "shape": lambda: fs(x, x[:1]),
        "rank3": lambda: fs(x[0], x[0]),
        "kernel_len": lambda: fs(x, x, kernel_size=(3, 3, 3)),
        "sigma_len": lambda: fs(x, x, sigma=(1.0, 1.0, 1.0)),
        "exclusive": lambda: fs(x, x, return_full_image=True, return_contrast_sensitivity=True),
        "kernel_even": lambda: fs(x, x, kernel_size=4),
        "kernel_even_before_sigma": lambda: fs(x, x, kernel_size=4, sigma=-1.0),
        "sigma_negative": lambda: fs(x, x, sigma=-1.0),
        "reflect_pad": lambda: fs(x[..., :5, :5], x[..., :5, :5], data_range=1.0),
        "reflect_pad_3d": lambda: fs(v[:, :, :3], v[:, :, :3], kernel_size=(3, 3, 3), data_range=1.0),
        "conv_size_3d": lambda: fs(v, v, data_range=1.0, kernel_size=(3, 3, 3), sigma=(0.5, 0.5, 3.0)),
        "empty_batch_none": lambda: fs(x[:0], x[:0]),
        "empty_batch_range": lambda: fs(x[:0], x[:0], data_range=1.0),
        "no_channels": lambda: fs(x[:, :0], x[:, :0], data_range=1.0),
        "no_channels_3d": lambda: fs(v[:, :0], v[:, :0], data_range=1.0, kernel_size=3),
        "no_channels_ms": lambda: fm(torch.rand(1, 0, 180, 180), torch.rand(1, 0, 180, 180), data_range=1.0),
        "int_inputs": lambda: fs((x * 10).long(), (x * 10).long()),
        "bool_inputs": lambda: fs(x > 0.5, x > 0.5),
        "bool_inputs_range": lambda: fs(x > 0.5, x > 0.5, data_range=1.0),
        "ms_betas_type": lambda: fm(big, big, betas=[0.5, 0.5]),
        "ms_betas_float": lambda: fm(big, big, betas=(1, 2)),
        "ms_normalize": lambda: fm(big, big, normalize="x"),
        "ms_small": lambda: fm(x, x),
        "ms_height": lambda: fm(big, big),
        "ms_width": lambda: fm(torch.rand(1, 1, 180, 64), torch.rand(1, 1, 180, 64)),
        "ms_late_reflect": lambda: fm(torch.rand(1, 1, 2, 64, 64), torch.rand(1, 1, 2, 64, 64), betas=(0.5, 0.5),
                                      data_range=1.0, kernel_size=3, sigma=0.3),
        "cls_reduction": lambda: S.StructuralSimilarityIndexMeasure(reduction="mean"),
        "ms_cls_reduction": lambda: S.MultiScaleStructuralSimilarityIndexMeasure(reduction="mean"),
        "ms_cls_kernel_type": lambda: S.MultiScaleStructuralSimilarityIndexMeasure(kernel_size=3.0),
        "ms_cls_kernel_len": lambda: S.MultiScaleStructuralSimilarityIndexMeasure(kernel_size=(3,)),
        "ms_cls_betas": lambda: S.MultiScaleStructuralSimilarityIndexMeasure(betas=[0.5]),
        "ms_cls_normalize": lambda: S.MultiScaleStructuralSimilarityIndexMeasure(normalize="x"),
    }


def ssim_golden() -> tuple[dict, dict]:
    sys.path.insert(0, ROOT)
    from tests import ssim_cases as sc

    F = importlib.import_module("torchmetrics.functional.image.ssim")  # noqa: N806
    S = importlib.import_module("torchmetrics.image.ssim")  # noqa: N806
    out = {}
    for case in sc.cases():
        out.update(sc.run_case(case, F, S))
    for level, noise in OFFSETS:
        p, t = sc.offset_pair(level, noise)
        for dt, tag in ((torch.float64, "f64"), (torch.float32, "f32")):
            r = F.structural_similarity_index_measure(torch.from_numpy(p).to(dt), torch.from_numpy(t).to(dt),
                                                      data_range=1.0, reduction="none")
            out[f"offset_{level:g}/{tag}"] = r.numpy()
    errors = {}
    for name, call in error_calls(F, S).items():
        try:
            call()
        except Exception as e:  # noqa: BLE001
            errors[name] = [type(e).__name__, str(e)]
        else:
            errors[name] = None
    return out, errors


if __name__ == "__main__":
    import warnings

    warnings.simplefilter("ignore")
    sys.path.insert(0, os.path.join(HERE, "_standins"))
    sys.path.insert(0, "/root/reference/src")
    data, errors = ssim_golden()
    path = os.path.join(HERE, "ssim.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB,", len(data), "arrays")
    surface = {"surface": ssim_surface("torchmetrics"), "states": ssim_states("torchmetrics"), "errors": errors}
    with open(os.path.join(HERE, "ssim_surface.json"), "w") as fh:
        json.dump(surface, fh, indent=0, sort_keys=True)
    print("wrote ssim_surface.json")
