"""Generate tests/golden/vif_uqi.npz and tests/golden/vif_uqi_surface.json from the UNMODIFIED reference (TorchMetrics
under /root/reference), CPU tensors.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_vif_uqi.py

Same import set-up as make_golden_ssim.py.  Every case of tests/vif_uqi_cases.py goes through the reference functional on
its first batch and the reference class over both batches, in the case's dtype.  The offset workloads (a ramp at level 0,
100 and 1000 plus noise) are recorded in float64 and in the reference's float32.  The json holds the signatures, the
class attributes, the state registries and the reference's error types and messages.
"""
from __future__ import annotations

import importlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from tests.golden.make_golden_ssim import ATTRS, _signature  # noqa: E402

OFFSETS = ((0.0, 1e-2), (100.0, 1e-2), (1000.0, 1e-2))
MODULES = {"vif": ("VisualInformationFidelity", "visual_information_fidelity"),
           "uqi": ("UniversalImageQualityIndex", "universal_image_quality_index")}


def modules(pkg: str) -> dict:
    return {k: (importlib.import_module(f"{pkg}.functional.image.{k}"), importlib.import_module(f"{pkg}.image.{k}"))
            for k in MODULES}


def surface(pkg: str) -> dict:
    out = {}
    for k, (F, S) in modules(pkg).items():  # noqa: N806
        cls_name, fn_name = MODULES[k]
        cls = getattr(S, cls_name)
        out[f"image.{cls_name}"] = {"init": _signature(cls.__init__), "update": _signature(cls.update),
                                    "compute": _signature(cls.compute),
                                    "attrs": {a: repr(getattr(cls, a, None)) for a in ATTRS}}
        out[f"functional.image.{fn_name}"] = {"call": _signature(getattr(F, fn_name))}
    return out


def states(pkg: str) -> dict:
    mods = modules(pkg)
    out = {}
    for label, make in (("vif", lambda: mods["vif"][1].VisualInformationFidelity()),
                        ("uqi_mean", lambda: mods["uqi"][1].UniversalImageQualityIndex()),
                        ("uqi_sum", lambda: mods["uqi"][1].UniversalImageQualityIndex(reduction="sum")),
                        ("uqi_none", lambda: mods["uqi"][1].UniversalImageQualityIndex(reduction="none"))):
        m = make()
        out[label] = {k: {"default": [list(v.shape), str(v.dtype)] if isinstance(v, torch.Tensor) else repr(v),
                          "reduce": getattr(m._reductions[k], "__name__", None), "persistent": m._persistent[k]}
                      for k, v in m._defaults.items()}
    return out


def error_calls(mods: dict) -> dict:
    """name -> call for either package's modules (CPU inputs: every one of these errors is raised before any data is
    read)."""
    (fv, sv), (fu, su) = mods["vif"], mods["uqi"]
    v, fn = torch.rand(2, 3, 41, 41), fv.visual_information_fidelity
    x, fq = torch.rand(2, 3, 16, 16), fu.universal_image_quality_index
    return {
        "vif_small_preds": lambda: fn(v[..., :40, :], v),
        "vif_small_target": lambda: fn(v, v[..., :40]),
        "vif_rank3": lambda: fn(torch.rand(3, 41, 41), torch.rand(3, 41, 41)),
        "vif_rank5": lambda: fn(torch.rand(1, 1, 2, 41, 41), torch.rand(1, 1, 2, 41, 41)),
        "vif_no_channels": lambda: fn(v[:, :0], v[:, :0]),
        "vif_int": lambda: fn((v * 10).long(), (v * 10).long()),
        "vif_bool": lambda: fn(v > 0.5, v > 0.5),
        "vif_mixed_target_f64": lambda: fn(v, v.double()),
        "vif_mixed_preds_f64": lambda: fn(v.double(), v),
        "vif_cls_scale0": lambda: sv.VisualInformationFidelity().update(torch.rand(1, 1, 16, 30), torch.rand(1, 1, 16, 30)),
        "vif_cls_scale1": lambda: sv.VisualInformationFidelity().update(torch.rand(1, 1, 20, 20), torch.rand(1, 1, 20, 20)),
        "vif_cls_scale2": lambda: sv.VisualInformationFidelity().update(torch.rand(1, 1, 30, 30), torch.rand(1, 1, 30, 30)),
        "vif_cls_scale3": lambda: sv.VisualInformationFidelity().update(torch.rand(1, 1, 36, 40), torch.rand(1, 1, 36, 40)),
        "vif_cls_sigma_type": lambda: sv.VisualInformationFidelity(sigma_n_sq="a"),
        "vif_cls_sigma_negative": lambda: sv.VisualInformationFidelity(sigma_n_sq=-1.0),
        "uqi_mixed": lambda: fq(x, x.double()),
        "uqi_shape": lambda: fq(x, x[:1]),
        "uqi_rank3": lambda: fq(x[0], x[0]),
        "uqi_kernel_len": lambda: fq(x, x, kernel_size=(3, 3, 3)),
        "uqi_sigma_len": lambda: fq(x, x, sigma=(1.0,)),
        "uqi_kernel_even": lambda: fq(x, x, kernel_size=(4, 3)),
        "uqi_sigma_negative": lambda: fq(x, x, sigma=(1.0, -1.0)),
        "uqi_reflect_pad": lambda: fq(x[..., :5, :5], x[..., :5, :5]),
        "uqi_conv_size": lambda: fq(x[..., :8, :], x[..., :8, :], kernel_size=(11, 3)),
        "uqi_empty_batch": lambda: fq(x[:0], x[:0]),
        "uqi_no_channels": lambda: fq(x[:, :0], x[:, :0]),
        "uqi_int": lambda: fq((x * 10).long(), (x * 10).long()),
        "uqi_bool": lambda: fq(x > 0.5, x > 0.5),
        "uqi_reduction": lambda: fq(x, x, reduction="mean"),
        "uqi_cls_reduction": lambda: su.UniversalImageQualityIndex(reduction="mean"),
        "uqi_cls_mixed": lambda: su.UniversalImageQualityIndex().update(x, x.double()),
    }


def golden() -> tuple[dict, dict]:
    from tests import vif_uqi_cases as vc

    mods = modules("torchmetrics")
    out = {}
    for case in vc.cases():
        out.update(vc.run_case(case, *mods["vif"], *mods["uqi"]))
    for level, noise in OFFSETS:
        p, t = vc.offset_pair(level, noise)
        for dt, tag in ((torch.float64, "f64"), (torch.float32, "f32")):
            pt, tt = torch.from_numpy(p).to(dt), torch.from_numpy(t).to(dt)
            out[f"offset_{level:g}/vif_{tag}"] = mods["vif"][0].visual_information_fidelity(pt, tt).numpy()
            out[f"offset_{level:g}/uqi_{tag}"] = mods["uqi"][0].universal_image_quality_index(pt, tt).numpy()
    errors = {}
    for name, call in error_calls(mods).items():
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
    data, errors = golden()
    path = os.path.join(HERE, "vif_uqi.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB,", len(data), "arrays")
    doc = {"surface": surface("torchmetrics"), "states": states("torchmetrics"), "errors": errors}
    with open(os.path.join(HERE, "vif_uqi_surface.json"), "w") as fh:
        json.dump(doc, fh, indent=0, sort_keys=True)
    print("wrote vif_uqi_surface.json")
