"""Generate tests/golden/exact_curves.npz from the UNMODIFIED reference (TorchMetrics under /root/reference), CPU tensors.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_exact_curves.py

Same import set-up as make_golden.py.  Every set is an input whose exact-mode result does not depend on the order the
reference's argsort (`stable=False`) picks inside a tie, so the golden is reproducible byte for byte:
  * `clf/*`: `_binary_clf_curve` on NaN runs whose members share one label, on runs of +inf and of -inf (same label within
    each run), on NaN mixed with +-inf, and on int64 targets at and above 2^31 with pos_label 1;
  * `bin/*`: binary ROC, PR curve, AUROC and AP through the functionals with NaN runs (validate_args=False);
  * `ml/*`: multilabel ROC / PR / AUROC / AP with uint8, int8 and int16 targets and an `ignore_index` that wraps in the
    target's dtype (uint8 257 and -1, int8 255, int16 65535);
  * `mc/*`: multiclass AUROC / AP / ROC with int64 targets 2^32 + c (validate_args=False): no class holds them.
tests/test_oracle_exact_curves.py replays them through oracle/exact_curves.py.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "_standins"))
sys.path.insert(0, "/root/reference/src")
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import torchmetrics.functional.classification as F  # noqa: E402
import torchmetrics.functional.classification.precision_recall_curve  # noqa: E402,F401

prc = sys.modules["torchmetrics.functional.classification.precision_recall_curve"]
NAN, INF = float("nan"), float("inf")


def clf_cases():
    """name -> (preds, target): every NaN / +inf / -inf run holds one label only."""
    g = torch.Generator().manual_seed(7)
    out = {
        "nan_pos": (torch.tensor([NAN, 0.5, NAN, 0.5, 0.25, NAN]), torch.tensor([1, 0, 1, 1, 0, 1])),
        "nan_neg": (torch.tensor([NAN, 0.5, NAN, 0.5, 0.25, NAN]), torch.tensor([0, 0, 0, 1, 1, 0])),
        "inf_runs": (torch.tensor([INF, INF, 1.0, -INF, 0.0, -INF, INF]), torch.tensor([1, 1, 0, 0, 1, 0, 1])),
        "nan_inf": (torch.tensor([-INF, NAN, INF, NAN, 0.5, -INF, INF]), torch.tensor([1, 0, 1, 0, 1, 1, 1])),
        "all_nan": (torch.full((5,), NAN), torch.tensor([1, 1, 1, 1, 1])),
    }
    p = torch.rand(300, generator=g)
    t = torch.randint(0, 2, (300,), generator=g)
    p[t == 1] = torch.where(torch.rand(int((t == 1).sum()), generator=g) < 0.2, NAN, p[t == 1])
    p[t == 0] = torch.where(torch.rand(int((t == 0).sum()), generator=g) < 0.1, -INF, p[t == 0])
    out["rand_nan_pos_ninf_neg"] = (p, t)
    for dt in (torch.float16, torch.bfloat16, torch.float64):
        out[f"nan_pos_{str(dt)[6:]}"] = (out["nan_pos"][0].to(dt), out["nan_pos"][1])
    out["big_target"] = (torch.rand(64, generator=g), torch.randint(0, 2, (64,), generator=g) * (2**32 + 1))
    out["big_target_2e31"] = (torch.rand(64, generator=g), torch.where(torch.arange(64) % 3 == 0, 2**31, 1))
    return out


def ml_cases():
    """name -> (preds [N, 3], target [N, 3] of a small dtype, ignore_index)."""
    g = torch.Generator().manual_seed(11)
    out = {}
    for tdt, vals, ign in ((torch.uint8, [0, 1, 255], 257), (torch.uint8, [0, 1, 255], -1), (torch.int8, [0, 1, -1], 255),
                           (torch.int16, [0, 1, -1], 65535)):
        p = torch.rand(97, 3, generator=g)
        t = torch.tensor(vals)[torch.randint(0, 3, (97, 3), generator=g)].to(tdt)
        p[::7, 1] = NAN
        t[::7, 1] = 1  # a NaN run of positives only
        out[f"{str(tdt)[6:]}_{ign}"] = (p, t, ign)
    return out


def main() -> None:
    out: dict = {}
    for name, (p, t) in clf_cases().items():
        fps, tps, thr = prc._binary_clf_curve(p, t, pos_label=1)
        out[f"clf/{name}/preds"] = p.float().numpy() if p.dtype == torch.bfloat16 else p.numpy()
        out[f"clf/{name}/target"] = t.numpy()
        out[f"clf/{name}/fps"] = fps.numpy()
        out[f"clf/{name}/tps"] = tps.numpy()
        out[f"clf/{name}/thr"] = thr.float().numpy() if thr.dtype == torch.bfloat16 else thr.numpy()
        if p.dtype == torch.float32 and name.startswith(("nan", "rand", "all")):
            kw = dict(validate_args=False)
            out[f"bin/{name}/auroc"] = F.binary_auroc(p, t, **kw).numpy()
            out[f"bin/{name}/ap"] = F.binary_average_precision(p, t, **kw).numpy()
            for k, v in zip(("fpr", "tpr", "thr"), F.binary_roc(p, t, **kw)):
                out[f"bin/{name}/roc_{k}"] = v.numpy()
            for k, v in zip(("p", "r", "thr"), F.binary_precision_recall_curve(p, t, **kw)):
                out[f"bin/{name}/prc_{k}"] = v.numpy()
    for name, (p, t, ign) in ml_cases().items():
        out[f"ml/{name}/preds"] = p.numpy()
        out[f"ml/{name}/target"] = t.numpy()
        out[f"ml/{name}/ignore"] = np.int64(ign)
        kw = dict(num_labels=3, ignore_index=ign, validate_args=False)
        out[f"ml/{name}/auroc"] = F.multilabel_auroc(p, t, average="none", **kw).numpy()
        out[f"ml/{name}/ap"] = F.multilabel_average_precision(p, t, average="none", **kw).numpy()
        for k, vs in zip(("fpr", "tpr", "thr"), F.multilabel_roc(p, t, **kw)):
            for i, v in enumerate(vs):
                out[f"ml/{name}/roc_{k}{i}"] = v.numpy()
        for k, vs in zip(("p", "r", "thr"), F.multilabel_precision_recall_curve(p, t, **kw)):
            for i, v in enumerate(vs):
                out[f"ml/{name}/prc_{k}{i}"] = v.numpy()
    g = torch.Generator().manual_seed(13)
    p = torch.rand(200, 4, generator=g)
    t = torch.randint(0, 4, (200,), generator=g)
    t[::5] += 2**32  # 2^32 + c: equal to no class in 64 bits
    out["mc/big/preds"] = p.numpy()
    out["mc/big/target"] = t.numpy()
    kw = dict(num_classes=4, average="none", validate_args=False)
    out["mc/big/auroc"] = F.multiclass_auroc(p, t, **kw).numpy()
    out["mc/big/ap"] = F.multiclass_average_precision(p, t, **kw).numpy()
    for k, vs in zip(("fpr", "tpr", "thr"), F.multiclass_roc(p, t, num_classes=4, validate_args=False)):
        for i, v in enumerate(vs):
            out[f"mc/big/roc_{k}{i}"] = v.numpy()
    path = os.path.join(HERE, "exact_curves.npz")
    np.savez_compressed(path, **{k: out[k] for k in sorted(out)})
    print(f"wrote {len(out)} arrays to {path}")


if __name__ == "__main__":
    main()
