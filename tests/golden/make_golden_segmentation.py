"""Generate tests/golden/segmentation.npz and tests/golden/segmentation_surface.json from the UNMODIFIED reference
(TorchMetrics under /root/reference), CPU tensors.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_segmentation.py

Same import set-up as make_golden.py.  Every case feeds one or more batches through a reference class and stores the
inputs, the class states, `compute()` and the functional's result on the first batch.  The json holds the public surface
(parameters and defaults, class metadata) and the state registry of the three classes; `seg_surface` / `seg_states` are
also what tests/test_segmentation_surface.py runs on this package.
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
KINDS = ("MeanIoU", "DiceScore", "GeneralizedDiceScore")
FUNCTIONALS = ("mean_iou", "dice_score", "generalized_dice_score")
AVERAGES = ("micro", "macro", "weighted", "none", None)
WEIGHTS = ("square", "simple", "linear")
DTYPES = {torch.int64: 0, torch.bool: 1, torch.uint8: 2, torch.float32: 3, torch.float16: 4, torch.int32: 5}
ATTRS = ("higher_is_better", "is_differentiable", "full_state_update", "plot_lower_bound", "plot_upper_bound")
# constructor variants of the state registry
VARIANTS = {"default": dict(num_classes=5), "no_bg": dict(num_classes=5, include_background=False),
            "per_class": dict(num_classes=5, per_class=True), "per_class_no_bg": dict(num_classes=5, per_class=True,
                                                                                       include_background=False)}


def _signature(fn):
    sig = inspect.signature(fn)
    return [[n, "<required>" if p.default is inspect.Parameter.empty else repr(p.default)] for n, p in sig.parameters.items()
            if n != "self"]


def seg_surface(pkg: str) -> dict:
    mod = importlib.import_module(f"{pkg}.segmentation")
    fmod = importlib.import_module(f"{pkg}.functional.segmentation")
    out = {"segmentation.__all__": sorted(mod.__all__), "functional.segmentation.__all__": sorted(fmod.__all__)}
    for name in KINDS:
        cls = getattr(mod, name)
        out[f"segmentation.{name}"] = {"init": _signature(cls.__init__), "update": _signature(cls.update),
                                       "compute": _signature(cls.compute),
                                       "attrs": {a: repr(getattr(cls, a, None)) for a in ATTRS}}
    for name in FUNCTIONALS:
        out[f"functional.segmentation.{name}"] = {"call": _signature(getattr(fmod, name))}
    return out


def seg_states(pkg: str) -> dict:
    mod = importlib.import_module(f"{pkg}.segmentation")
    out = {}
    for name in KINDS:
        for variant, kwargs in VARIANTS.items():
            if "per_class" in kwargs and name == "DiceScore":
                kwargs = {k: v for k, v in kwargs.items() if k != "per_class"}
            m = getattr(mod, name)(**kwargs)
            out[f"{name}[{variant}]"] = {
                k: {"default": "list" if isinstance(v, list) else [list(v.shape), str(v.dtype)],
                    "reduce": getattr(m._reductions[k], "__name__", None) if m._reductions[k] is not None else None,
                    "persistent": m._persistent[k]} for k, v in m._defaults.items()}
    return out


def np_of(t: torch.Tensor) -> np.ndarray:
    return t.float().numpy() if t.dtype in (torch.float16, torch.bfloat16) else t.numpy()


def label_map(g, n, shape, c, coherent: bool) -> torch.Tensor:
    """Random labels; `coherent` maps are blocks of 4 x 4 (the last two axes) of one class."""
    if not coherent or len(shape) < 2:
        return torch.randint(0, c, (n, *shape), generator=g)
    small = torch.randint(0, c, (n, *shape[:-2], (shape[-2] + 3) // 4, (shape[-1] + 3) // 4), generator=g)
    big = small.repeat_interleave(4, -2).repeat_interleave(4, -1)
    return big[..., : shape[-2], : shape[-1]].contiguous()


def one_hot_of(labels: torch.Tensor, c: int, dtype: torch.dtype, layout: int) -> torch.Tensor:
    x = torch.nn.functional.one_hot(labels, c).movedim(-1, 1).to(dtype)
    return x if layout == 1 else x.contiguous()


def segmentation_golden() -> dict:
    from torchmetrics import segmentation as S  # noqa: N812
    from torchmetrics.functional import segmentation as F  # noqa: N812

    g = torch.Generator().manual_seed(1515)
    out = {}
    case = 0

    def put(kind, batches, num_classes, include_background, option, index, layout=0):
        nonlocal case
        key = f"case{case}"
        kw = dict(num_classes=num_classes, include_background=include_background,
                  input_format="index" if index else "one-hot")
        if kind == 0:
            m, f = S.MeanIoU(per_class=bool(option), **kw), lambda p, t: F.mean_iou(p, t, per_class=bool(option), **kw)
        elif kind == 1:
            m, f = S.DiceScore(average=AVERAGES[option], **kw), lambda p, t: F.dice_score(p, t, average=AVERAGES[option], **kw)
        else:
            wt, pc = WEIGHTS[option % 3], option >= 3
            m = S.GeneralizedDiceScore(per_class=pc, weight_type=wt, **kw)
            f = lambda p, t: F.generalized_dice_score(p, t, per_class=pc, weight_type=wt, **kw)  # noqa: E731
        for b, (p, t) in enumerate(batches):
            m.update(p, t)
            out[f"{key}/preds{b}"], out[f"{key}/target{b}"] = np_of(p.contiguous()), np_of(t.contiguous())
        if kind == 0:
            out[f"{key}/score"], out[f"{key}/num_batches"] = m.score.numpy(), m.num_batches.numpy()
        elif kind == 1:
            for s in ("numerator", "denominator", "support"):
                out[f"{key}/{s}"] = np_of(torch.cat(getattr(m, s)))
        else:
            out[f"{key}/score"], out[f"{key}/samples"] = m.score.numpy(), m.samples.numpy()
        out[f"{key}/compute"] = np_of(m.compute())
        out[f"{key}/functional"] = np_of(f(*batches[0]))
        out[f"{key}/meta"] = np.array([kind, int(index), num_classes, int(include_background), option, len(batches),
                                       DTYPES[batches[0][0].dtype], layout])
        case += 1

    # index inputs: [N, d], [N, H, W], [N, D, H, W]; coherent and uniform maps; every option of every metric
    shapes = ((40,), (8, 12), (3, 5, 6))
    for kind, options in ((0, (0, 1)), (1, range(5)), (2, range(6))):
        for opt in options:
            for si, shape in enumerate(shapes):
                for bg in (True, False):
                    c = (5, 3, 19)[(opt + si) % 3]
                    batches = [(label_map(g, 3, shape, c, coherent=b % 2 == 0), label_map(g, 3, shape, c, coherent=b % 2 == 1))
                               for b in range(2)]
                    if kind == 2 and (opt + si) % 2 == 0:  # some classes missing from some samples' targets
                        batches[0][1].clamp_(max=c // 2)
                    put(kind, batches, c, bg, opt, True)
    # one-hot inputs: dtypes, planar and channels-last, non-binary uint8 (& against *), [N, C, d] .. [N, C, D, H, W]
    for kind, options in ((0, (0, 1)), (1, (0, 1, 2, 3)), (2, (0, 1, 5))):
        for dtype in (torch.bool, torch.uint8, torch.int64, torch.float32, torch.float16):
            if kind == 0 and dtype.is_floating_point:
                continue
            for layout in (0, 1):
                for opt in options:
                    shape = ((16,), (6, 7), (2, 3, 4))[(opt + layout) % 3]
                    c = 4
                    bg = (opt + layout) % 2 == 0
                    batches = []
                    for b in range(2):
                        p = one_hot_of(label_map(g, 3, shape, c, True), c, dtype, layout)
                        t = one_hot_of(label_map(g, 3, shape, c, False), c, dtype, layout)
                        batches.append((p, t))
                    put(kind, batches, c, bg, opt, False, layout)
    # non-binary uint8 values: `&` and `*` differ, and products wrap
    for kind, opt in ((0, 1), (1, 3), (2, 3)):
        p = torch.randint(0, 256, (2, 3, 5, 5), generator=g, dtype=torch.uint8)
        t = torch.randint(0, 256, (2, 3, 5, 5), generator=g, dtype=torch.uint8)
        put(kind, [(p, t)], 3, True, opt, False)
    # GeneralizedDice with N != C' and classes absent from some samples (the flat-index weight fill)
    for opt in range(6):
        t = label_map(g, 5, (6, 6), 3, True)
        t[1] = 0
        t[3] = 2
        put(2, [(label_map(g, 5, (6, 6), 3, False), t)], 3, bool(opt % 2), opt, True)
    # single-class and all-background batches
    z = torch.zeros(2, 8, 8, dtype=torch.long)
    put(1, [(z, z)], 4, False, 3, True)
    put(0, [(z, torch.full_like(z, 2))], 4, True, 1, True)

    # the reference's errors (CPU): (kind, preds, target, num_classes, input_format) -> exception type and message
    errors = {}

    def err(name, fn):
        try:
            fn()
        except Exception as e:  # noqa: BLE001
            errors[name] = [type(e).__name__, str(e)]

    lab = torch.randint(0, 4, (2, 5, 5), generator=g)
    neg, big = lab.clone(), lab.clone()
    neg[0, 1, 1], big[1, 2, 2] = -1, 4
    err("preds_negative", lambda: F.dice_score(neg, lab, 4, input_format="index"))
    err("preds_too_large", lambda: F.dice_score(big, lab, 4, input_format="index"))
    err("target_negative", lambda: F.dice_score(lab, neg, 4, input_format="index"))
    err("target_too_large", lambda: F.dice_score(lab, big, 4, input_format="index"))
    both = neg.clone()
    both[1, 2, 2] = 4
    err("preds_both", lambda: F.mean_iou(both, big, 4, input_format="index"))
    err("preds_large_target_negative", lambda: F.generalized_dice_score(big, neg, 4, input_format="index"))
    err("int32_index", lambda: F.dice_score(lab.int(), lab.int(), 4, input_format="index"))
    err("float_mean_iou", lambda: F.mean_iou(torch.rand(2, 3, 4, 4), torch.rand(2, 3, 4, 4), 3))
    err("shape", lambda: F.dice_score(lab, lab[:1], 4, input_format="index"))
    err("dice_2d", lambda: F.dice_score(torch.ones(2, 3, dtype=torch.long), torch.ones(2, 3, dtype=torch.long), 3))
    for name, fn in (("num_classes", lambda: S.MeanIoU(0)), ("input_format", lambda: S.DiceScore(3, input_format="x")),
                     ("average", lambda: S.DiceScore(3, average="samples")),
                     ("weight_type", lambda: S.GeneralizedDiceScore(3, weight_type="cubic")),
                     ("per_class", lambda: S.MeanIoU(3, per_class=1)),
                     ("include_background", lambda: S.GeneralizedDiceScore(3, include_background=None))):
        err(name, fn)
    out["n_cases"] = np.array(case)
    return out, errors


if __name__ == "__main__":
    import warnings

    warnings.simplefilter("ignore")
    sys.path.insert(0, os.path.join(HERE, "_standins"))
    sys.path.insert(0, "/root/reference/src")
    data, errors = segmentation_golden()
    path = os.path.join(HERE, "segmentation.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB,", int(data["n_cases"]), "cases")
    surface = {"surface": seg_surface("torchmetrics"), "states": seg_states("torchmetrics"), "errors": errors}
    with open(os.path.join(HERE, "segmentation_surface.json"), "w") as fh:
        json.dump(surface, fh, indent=0, sort_keys=True)
    print("wrote segmentation_surface.json")
