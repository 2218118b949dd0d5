"""Generate tests/golden/hausdorff.npz and tests/golden/hausdorff_surface.json from the UNMODIFIED reference (TorchMetrics
under /root/reference), CPU tensors.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_hausdorff.py

Same import set-up as make_golden.py.  Every case of tests/hausdorff_cases.py goes through the reference functional on
its first batch and the reference class over both batches (its states and `compute()`).  Square images only: the
reference scatters its distance transform with the column count as the row stride.  The json holds the signatures, the
class attributes, the state registry and the reference's error messages.
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


def _signature(fn):
    sig = inspect.signature(fn)
    return [[n, "<required>" if p.default is inspect.Parameter.empty else repr(p.default)] for n, p in sig.parameters.items()
            if n != "self"]


def hd_surface(pkg: str) -> dict:
    cls = importlib.import_module(f"{pkg}.segmentation.hausdorff_distance").HausdorffDistance
    fn = importlib.import_module(f"{pkg}.functional.segmentation.hausdorff_distance").hausdorff_distance
    return {"segmentation.HausdorffDistance": {"init": _signature(cls.__init__), "update": _signature(cls.update),
                                               "compute": _signature(cls.compute),
                                               "attrs": {a: repr(getattr(cls, a, None)) for a in ATTRS}},
            "functional.segmentation.hausdorff_distance": {"call": _signature(fn)}}


def hd_states(pkg: str) -> dict:
    cls = importlib.import_module(f"{pkg}.segmentation.hausdorff_distance").HausdorffDistance
    m = cls(num_classes=3)
    return {k: {"default": [list(v.shape), str(v.dtype)], "reduce": getattr(m._reductions[k], "__name__", None),
                "persistent": m._persistent[k]} for k, v in m._defaults.items()}


def error_calls(F, S):  # noqa: N803
    """name -> call, for the functional module F and the class module S of either package (CPU inputs)."""
    ok = torch.ones(2, 3, 6, 6, dtype=torch.int64)
    ok[:, :, 2:4, 2:4] = 0
    nb_p, nb_t = ok.clone(), ok.clone()
    nb_p[1, 1, 0, 0], nb_t[0, 2, 5, 5] = 2, -1
    empty = ok.clone()
    empty[0, 2] = 0
    late_nb = empty.clone()  # pair (0, 2) empty on both sides, then a non-binary target in pair (1, 1)
    late_nb[1, 1, 3, 3] = 3
    early_nb = ok.clone()  # a non-binary preds value in pair (0, 1), then pair (1, 2) empty on both sides
    early_nb[0, 1, 0, 0] = 2
    early_nb[1, 2] = 0
    late_empty = ok.clone()
    late_empty[1, 2] = 0
    lab = torch.randint(0, 3, (2, 6, 6), generator=torch.Generator().manual_seed(0))
    neg, big = lab.clone(), lab.clone()
    neg[1, 0, 0], big[0, 1, 1] = -1, 3
    return {
        "preds_not_binary": lambda: F.hausdorff_distance(nb_p, ok, 3),
        "target_not_binary": lambda: F.hausdorff_distance(ok, nb_t, 3),
        "both_empty": lambda: F.hausdorff_distance(empty, empty, 3),
        "empty_before_not_binary": lambda: F.hausdorff_distance(empty, late_nb, 3, include_background=True),
        "not_binary_before_empty": lambda: F.hausdorff_distance(early_nb, late_empty, 3),
        "preds_negative": lambda: F.hausdorff_distance(neg, lab, 3, input_format="index"),
        "target_too_large": lambda: F.hausdorff_distance(lab, big, 3, input_format="index"),
        "int32_index": lambda: F.hausdorff_distance(lab.int(), lab.int(), 3, input_format="index"),
        "float_one_hot": lambda: F.hausdorff_distance(ok.float(), ok, 3),
        "half_target": lambda: F.hausdorff_distance(ok, ok.half(), 3),
        "spacing_tensor": lambda: F.hausdorff_distance(ok, ok, 3, spacing=torch.tensor([1.0, 2.0])),
        "spacing_len3": lambda: F.hausdorff_distance(ok, ok, 3, spacing=[1, 1, 1]),
        "rank3": lambda: F.hausdorff_distance(ok[..., None].expand(-1, -1, -1, -1, 3), ok[..., None].expand(-1, -1, -1, -1, 3), 3),
        "rank1": lambda: F.hausdorff_distance(ok[:, :, 0], ok[:, :, 0], 3),
        "shape": lambda: F.hausdorff_distance(ok, ok[:1], 3),
        "num_classes": lambda: S.HausdorffDistance(0),
        "include_background": lambda: S.HausdorffDistance(3, include_background=1),
        "metric": lambda: S.HausdorffDistance(3, distance_metric="cosine"),
        "spacing_type": lambda: S.HausdorffDistance(3, spacing=(1, 1)),
        "directed": lambda: S.HausdorffDistance(3, directed=None),
        "input_format": lambda: S.HausdorffDistance(3, input_format="x"),
    }


def hausdorff_golden() -> tuple[dict, dict]:
    sys.path.insert(0, ROOT)
    from tests import hausdorff_cases as hc
    F = importlib.import_module("torchmetrics.functional.segmentation.hausdorff_distance")  # noqa: N806
    S = importlib.import_module("torchmetrics.segmentation.hausdorff_distance")  # noqa: N806

    out = {}
    for case in hc.cases():
        name, kw = case["name"], case["kwargs"]
        (p0, t0), (p1, t1) = hc.tensors(case)
        out[f"{name}/functional"] = F.hausdorff_distance(p0, t0, **kw).numpy()
        m = S.HausdorffDistance(**kw)
        m.update(p0, t0)
        m.update(p1, t1)
        out[f"{name}/score"], out[f"{name}/total"] = m.score.numpy(), m.total.numpy()
        out[f"{name}/compute"] = m.compute().numpy()
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
    data, errors = hausdorff_golden()
    path = os.path.join(HERE, "hausdorff.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB,", len(data), "arrays")
    surface = {"surface": hd_surface("torchmetrics"), "states": hd_states("torchmetrics"), "errors": errors}
    with open(os.path.join(HERE, "hausdorff_surface.json"), "w") as fh:
        json.dump(surface, fh, indent=0, sort_keys=True)
    print("wrote hausdorff_surface.json")
