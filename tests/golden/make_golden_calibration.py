"""Generate tests/golden/calibration.npz from the UNMODIFIED reference (TorchMetrics under /root/reference), CPU tensors.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_calibration.py

Same import set-up as make_golden.py (the stand-in for the reference's missing `lightning_utilities`).  Every case stores
its inputs, the reference's states (confidences, accuracies) and `compute()` for the three norms.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "_standins"))
sys.path.insert(0, "/root/reference/src")

from torchmetrics.classification import BinaryCalibrationError, MulticlassCalibrationError  # noqa: E402
from torchmetrics.functional.classification import binary_calibration_error, multiclass_calibration_error  # noqa: E402
from torchmetrics.functional.classification.calibration_error import _ce_compute  # noqa: E402

DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2, torch.float64: 3}


def np_of(t: torch.Tensor) -> np.ndarray:
    """float16 / bfloat16 are stored widened to float32 (exact); the dtype code says what to narrow them back to."""
    return t.float().numpy() if t.dtype in (torch.float16, torch.bfloat16) else t.numpy()


def calibration_golden() -> dict:
    g = torch.Generator().manual_seed(1414)
    out = {}
    case = 0

    def put(kind, batches, n_bins, ignore_index, num_classes=0):
        nonlocal case
        key = f"case{case}"
        cls = (BinaryCalibrationError(n_bins=n_bins, ignore_index=ignore_index) if kind == "binary"
               else MulticlassCalibrationError(num_classes, n_bins=n_bins, ignore_index=ignore_index))
        for preds, target in batches:
            cls.update(preds, target)
        for b, (preds, target) in enumerate(batches):
            out[f"{key}/preds{b}"], out[f"{key}/target{b}"] = np_of(preds), target.numpy()
        conf, acc = torch.cat(cls.confidences), torch.cat(cls.accuracies)
        out[f"{key}/conf"], out[f"{key}/acc"] = np_of(conf), acc.numpy()
        for norm in ("l1", "l2", "max"):
            out[f"{key}/{norm}"] = np_of(_ce_compute(conf, acc, n_bins, norm).reshape(()).to(conf.dtype))
        out[f"{key}/meta"] = np.array([kind == "binary", len(batches), n_bins, -999 if ignore_index is None else ignore_index,
                                       num_classes, DTYPE_CODE[batches[0][0].dtype]])
        case += 1

    # docstring examples
    p = torch.tensor([0.25, 0.25, 0.55, 0.75, 0.75])
    t = torch.tensor([0, 0, 1, 1, 1])
    out["doc/binary"] = np.array([float(binary_calibration_error(p, t, n_bins=2, norm=n)) for n in ("l1", "l2", "max")])
    p = torch.tensor([[0.25, 0.20, 0.55], [0.55, 0.05, 0.40], [0.10, 0.30, 0.60], [0.90, 0.05, 0.05]])
    t = torch.tensor([0, 1, 2, 0])
    out["doc/multiclass"] = np.array([float(multiclass_calibration_error(p, t, num_classes=3, n_bins=3, norm=n))
                                      for n in ("l1", "l2", "max")])

    # multiclass: logits and probabilities, C in {2, 5, 1000}, n_bins in {1, 15, 100}, ignore_index in {None, -1, 0}
    for c in (2, 5, 1000):
        for logits in (True, False):
            for n_bins, ignore_index in ((15, None), (1, -1), (100, 0)):
                n = 300 if c < 1000 else 32
                x = torch.randn(n, c, generator=g) * 3
                preds = x if logits else torch.softmax(x, 1)
                target = torch.randint(0, c, (n,), generator=g)
                if ignore_index is not None:
                    target[::7] = ignore_index
                put("multiclass", [(preds, target)], n_bins, ignore_index, c)
    # only ignored rows hold scores outside [0, 1]: without them the batch is probabilities
    probs = torch.softmax(torch.randn(40, 4, generator=g), 1)
    target = torch.randint(0, 4, (40,), generator=g)
    probs[::5] = torch.randn(8, 4, generator=g) * 5
    target[::5] = -1
    put("multiclass", [(probs, target)], 10, -1, 4)
    # multidim [N, C, d] logits with ignore_index
    x = torch.randn(20, 6, 7, generator=g)
    target = torch.randint(0, 6, (20, 7), generator=g)
    target[:, ::3] = -1
    put("multiclass", [(x, target)], 15, -1, 6)
    # NaN rows in logits batches (the softmax of a NaN row is all NaN: confidence NaN, first index)
    x = torch.randn(50, 5, generator=g) * 2
    x[3, 2] = float("nan")
    x[17] = float("nan")
    put("multiclass", [(x, torch.randint(0, 5, (50,), generator=g))], 15, None, 5)
    # a class after several updates (mixed logits / probabilities batches)
    batches = []
    for i in range(4):
        x = torch.randn(100, 10, generator=g) * 2
        batches.append((x if i % 2 == 0 else torch.softmax(x, 1), torch.randint(0, 10, (100,), generator=g)))
    put("multiclass", batches, 15, None, 10)

    # binary: probabilities and logits, several dtypes, ignore_index, multidim
    for dtype in (torch.float32, torch.float16, torch.bfloat16, torch.float64):
        for logits in (True, False):
            for n_bins, ignore_index in ((15, None), (100, -1), (1, None)):
                x = torch.randn(500, generator=g, dtype=torch.float64) * 3
                preds = (x if logits else torch.sigmoid(x)).to(dtype)
                target = torch.randint(0, 2, (500,), generator=g)
                if ignore_index is not None:
                    target[::9] = ignore_index
                put("binary", [(preds, target)], n_bins, ignore_index)
    # confidences exactly on the boundaries and exactly 1.0 / 0.0
    for dtype in (torch.float32, torch.float16, torch.bfloat16, torch.float64):
        for n_bins in (15, 10, 4):
            bounds = torch.linspace(0, 1, n_bins + 1, dtype=dtype)
            preds = torch.cat([bounds, bounds, torch.ones(5, dtype=dtype), torch.zeros(3, dtype=dtype)])
            target = torch.randint(0, 2, (preds.numel(),), generator=g)
            put("binary", [(preds, target)], n_bins, None)
    # multidim binary, a class after several updates
    put("binary", [(torch.rand(8, 5, 3, generator=g), torch.randint(0, 2, (8, 5, 3), generator=g))], 15, None)
    put("binary", [(torch.rand(64, generator=g), torch.randint(0, 2, (64,), generator=g)),
                   (torch.randn(64, generator=g) * 4, torch.randint(0, 2, (64,), generator=g)),
                   (torch.rand(32, generator=g), torch.randint(0, 2, (32,), generator=g))], 15, None)
    # NaN scores in a logits batch: sigmoid keeps NaN, bucketize puts it in the last slot
    x = torch.randn(60, generator=g) * 3
    x[::11] = float("nan")
    put("binary", [(x, torch.randint(0, 2, (60,), generator=g))], 15, None)
    # perfectly calibrated l2: the reference returns the int64 `tensor(0)`
    preds = torch.tensor([0.0, 0.0, 1.0, 1.0])
    target = torch.tensor([0, 0, 1, 1])
    res = binary_calibration_error(preds, target, n_bins=4, norm="l2")
    out["l2zero/value"], out["l2zero/dtype_is_int64"] = res.numpy(), np.array(res.dtype == torch.int64)
    out["n_cases"] = np.array(case)
    return out


if __name__ == "__main__":
    data = calibration_golden()
    path = os.path.join(HERE, "calibration.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB,", len(data), "arrays")
