"""Generate tests/golden/panoptic.npz and tests/golden/panoptic_surface.json from the UNMODIFIED reference (TorchMetrics
under /root/reference), CPU tensors.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_panoptic.py

Same import set-up as make_golden.py.  Every case of tests/panoptic_cases.py goes through the reference class (the four
states and `compute()`) and its functional on the first batch; compute before any update is stored too.  The json holds
the functional signatures, the state registry of both classes and the reference's error messages.
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
KINDS = ("PanopticQuality", "ModifiedPanopticQuality")
FUNCTIONALS = ("panoptic_quality", "modified_panoptic_quality")
STATES = ("iou_sum", "true_positives", "false_positives", "false_negatives")
# constructor variants of the state registry
VARIANTS = {"things_stuffs": dict(things={0, 1}, stuffs={6, 7}), "things": dict(things=[3, 1, 2], stuffs=[]),
            "stuffs": dict(things=[], stuffs={5})}


def _signature(fn):
    sig = inspect.signature(fn)
    return [[n, "<required>" if p.default is inspect.Parameter.empty else repr(p.default)] for n, p in sig.parameters.items()
            if n != "self"]


def pq_surface(pkg: str) -> dict:
    fmod = importlib.import_module(f"{pkg}.functional.detection")
    return {f"functional.detection.{name}": {"call": _signature(getattr(fmod, name))} for name in FUNCTIONALS}


def pq_states(pkg: str) -> dict:
    mod = importlib.import_module(f"{pkg}.detection")
    out = {}
    for name in KINDS:
        for variant, kwargs in VARIANTS.items():
            m = getattr(mod, name)(**kwargs)
            out[f"{name}[{variant}]"] = {
                k: {"default": [list(v.shape), str(v.dtype)], "reduce": getattr(m._reductions[k], "__name__", None),
                    "persistent": m._persistent[k]} for k, v in m._defaults.items()}
    return out


def panoptic_golden() -> tuple[dict, dict]:
    sys.path.insert(0, ROOT)
    from tests import panoptic_cases as pc
    from torchmetrics import detection as D  # noqa: N812
    from torchmetrics.functional import detection as F  # noqa: N812

    out = {}
    for case in pc.golden_cases():
        key, kw = case["name"], dict(case["kwargs"])
        cls = D.ModifiedPanopticQuality if case["modified"] else D.PanopticQuality
        fn = F.modified_panoptic_quality if case["modified"] else F.panoptic_quality
        m = cls(case["things"], case["stuffs"], **kw)
        out[f"{key}/compute_empty"] = m.compute().numpy()
        for p, t in case["batches"]:
            m.update(p, t)
        for s in STATES:
            out[f"{key}/{s}"] = getattr(m, s).numpy()
        out[f"{key}/compute"] = m.compute().numpy()
        out[f"{key}/functional"] = fn(*case["batches"][0], case["things"], case["stuffs"], **kw).numpy()
    errors = {}

    def err(name, call):
        try:
            call()
        except Exception as e:  # noqa: BLE001
            errors[name] = [type(e).__name__, str(e)]

    p0, t0 = pc.inputs0()
    p1, t1 = pc.inputs1()
    err("unknown_preds", lambda: F.panoptic_quality(p1, t1, {0, 1}, {6, 7}))
    err("things_not_int", lambda: F.panoptic_quality(p0, t0, {0, 1.0}, {6, 7}))
    err("stuffs_not_int", lambda: F.panoptic_quality(p0, t0, {0, 1}, {6, "7"}))
    err("overlap", lambda: F.panoptic_quality(p0, t0, {0, 1}, {1, 7}))
    err("empty", lambda: D.PanopticQuality(set(), set()))
    err("preds_type", lambda: F.panoptic_quality(p0.numpy(), t0, {0, 1}, {6, 7}))
    err("target_type", lambda: F.panoptic_quality(p0, [1], {0, 1}, {6, 7}))
    err("shape", lambda: F.panoptic_quality(p0, t0[:, :3], {0, 1}, {6, 7}))
    err("dims", lambda: F.panoptic_quality(p0[0, 0], t0[0, 0], {0, 1}, {6, 7}))
    err("last_dim", lambda: F.panoptic_quality(p0[..., :1], t0[..., :1], {0, 1}, {6, 7}))
    return out, errors


if __name__ == "__main__":
    import warnings

    warnings.simplefilter("ignore")
    sys.path.insert(0, os.path.join(HERE, "_standins"))
    sys.path.insert(0, "/root/reference/src")
    data, errors = panoptic_golden()
    path = os.path.join(HERE, "panoptic.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB,", len(data), "arrays")
    surface = {"surface": pq_surface("torchmetrics"), "states": pq_states("torchmetrics"), "errors": errors}
    with open(os.path.join(HERE, "panoptic_surface.json"), "w") as fh:
        json.dump(surface, fh, indent=0, sort_keys=True)
    print("wrote panoptic_surface.json")
