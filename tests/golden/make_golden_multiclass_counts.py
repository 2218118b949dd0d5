"""Generate tests/golden/multiclass_counts.npz from the UNMODIFIED reference (TorchMetrics under /root/reference), CPU tensors.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_multiclass_counts.py

Same import set-up as make_golden.py.  The cases pin the counting chain behind the multiclass confusion matrix and stat
scores, for every target dtype (int8, uint8, int16, int32, int64, bool) and `ignore_index` in {None, -1, 0, C - 1, C} plus
the values ATen wraps to the target's dtype before comparing (257, -100 and -1 on uint8; 255 on int8; 65535 on int16).
Each set is counted by the reference's `multiclass_confusion_matrix` and `multiclass_stat_scores` (micro, none, top-k,
samplewise), with `validate_args=False`; whether `validate_args=True` raises is recorded too.  The scores are float32,
float16, bfloat16 or float64 `[N, C, X]` (and `[N * X, C]` for top-k), with rows holding NaN, +-inf, -0 / +0 and ties.
tests/test_oracle_multiclass_counts.py replays them through oracle/multiclass_counts.py.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "_standins"))
sys.path.insert(0, "/root/reference/src")

from torchmetrics.functional.classification import multiclass_confusion_matrix, multiclass_stat_scores  # noqa: E402

PREDS_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2, torch.float64: 3}
TARGET_DTYPES = [torch.int8, torch.uint8, torch.int16, torch.int32, torch.int64, torch.bool]
# value stored in the target for an ignore_index that lies outside the dtype's range: what ATen compares it as
WRAPPED = {torch.uint8: {257: 1, -100: 156, -1: 255}, torch.int8: {255: -1}, torch.int16: {65535: -1}}
N, X = 6, 4


def ignore_cases(dtype, c: int) -> list:
    """(ignore_index, stored value to plant or None)."""
    if dtype == torch.bool:
        return [(None, None), (0, None), (1, None)]
    out = [(None, None), (0, None), (c - 1, None), (c, c)]
    if dtype.is_signed:
        out.append((-1, -1))
    out += [(ign, stored) for ign, stored in WRAPPED.get(dtype, {}).items()]
    return out


def scores(shape, dtype, g: torch.Generator) -> torch.Tensor:
    """Random scores with NaN, +-inf, -0 / +0 and tied maxima planted along dim 1."""
    x = torch.randn(*shape, generator=g, dtype=torch.float64)
    flat = x.movedim(1, -1).reshape(-1, shape[1])  # one row per (n, x) position
    rows = flat.shape[0]
    special = torch.randperm(rows, generator=g)[: rows // 2]
    for i, r in enumerate(special.tolist()):
        kind = i % 6
        if kind == 0:
            flat[r, int(torch.randint(0, shape[1], (1,), generator=g))] = float("nan")
        elif kind == 1:
            flat[r] = float("-inf")
        elif kind == 2:
            flat[r] = 0.0
            flat[r, 0] = -0.0
        elif kind == 3:
            flat[r, -1] = flat[r, 0] = flat[r].abs().max() + 1  # tied maximum: first and last column
        elif kind == 4:
            flat[r, 1:] = float("inf")
        else:
            flat[r, :] = flat[r, 0]  # all equal
    x = flat.reshape(shape[0], *shape[2:], shape[1]).movedim(-1, 1)
    return x.to(dtype)


def np_of(t: torch.Tensor) -> np.ndarray:
    return t.float().numpy() if t.dtype in (torch.float16, torch.bfloat16) else t.numpy()


def multiclass_counts_golden() -> dict:
    g = torch.Generator().manual_seed(2025)
    out = {}
    case = 0
    for ti, tdtype in enumerate(TARGET_DTYPES):
        for c in ((2,) if tdtype == torch.bool else (3, 7)):
            for ign, stored in ignore_cases(tdtype, c):
                pdtype = list(PREDS_CODE)[case % 4]
                key = f"set{case}"
                p = scores((N, c, X), pdtype, g)
                pk = scores((N * X, c), pdtype, g)
                t = torch.randint(0, c, (N, X), generator=g)
                if stored is not None:
                    t[torch.rand(N, X, generator=g) < 0.25] = stored
                t = t.to(tdtype)
                tk = t.flatten()
                out[f"{key}/preds"], out[f"{key}/preds_topk"] = np_of(p), np_of(pk)
                out[f"{key}/target"] = t.numpy()
                out[f"{key}/meta"] = np.array([PREDS_CODE[pdtype], c, int(ign is not None), 0 if ign is None else ign])
                lab = torch.randint(0, c, (N, X), generator=g)
                out[f"{key}/labels"] = lab.numpy()
                out[f"{key}/confmat"] = multiclass_confusion_matrix(p, t, c, ignore_index=ign, validate_args=False).numpy()
                out[f"{key}/confmat_labels"] = multiclass_confusion_matrix(
                    lab, t, c, ignore_index=ign, validate_args=False).numpy()
                for avg in ("micro", "none"):
                    s = multiclass_stat_scores(p, t, c, average=avg, ignore_index=ign, validate_args=False)
                    out[f"{key}/stats_{avg}"] = s[..., :4].numpy()
                sw = multiclass_stat_scores(p, t, c, average="none", multidim_average="samplewise", ignore_index=ign,
                                            validate_args=False)
                out[f"{key}/stats_samplewise"] = sw[..., :4].numpy()
                if c >= 3:
                    s = multiclass_stat_scores(pk, tk, c, average="none", top_k=2, ignore_index=ign, validate_args=False)
                    out[f"{key}/stats_top2"] = s[..., :4].numpy()
                try:
                    multiclass_confusion_matrix(p, t, c, ignore_index=ign, validate_args=True)
                    raises = 0
                except RuntimeError:
                    raises = 1
                out[f"{key}/validate_raises"] = np.array(raises)
                case += 1
    out["n_sets"] = np.array(case)
    return out


if __name__ == "__main__":
    data = multiclass_counts_golden()
    path = os.path.join(HERE, "multiclass_counts.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB,", len(data), "arrays")
