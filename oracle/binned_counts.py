"""Oracle for the binned (fixed-threshold) curve state `[T, (C,) 2, 2]` (kernel K4, csrc/binned.cu).  TEST INFRASTRUCTURE
ONLY — see oracle/__init__.py.

Like oracle/binary_counts.py, this is the reference's own chain of torch ops, restated device-agnostically (on a GPU it runs
on the kernel's device, as the arbiter): the binary, multiclass (and micro) and multilabel format + update functions of
functional/classification/precision_recall_curve.py (:164-251, :430-533, :745-799), both of their update branches and the
size rule that picks one:

  * vectorized (binary `preds.numel() <= 50_000`, multiclass `preds.numel() * num_classes <= 1_000_000`, multilabel always):
    `preds.unsqueeze(-1) >= thresholds.unsqueeze(0)` compares in `torch.promote_types(score, threshold)`;
  * loop (above those sizes): `preds >= thresholds[i]` with a 0-dim threshold compares in the SCORE dtype, the threshold
    first rounded to it (double -> float -> half / bfloat16).

One departure from the letter of the multilabel format (:766-772): the reference writes the sentinel `-4 * L * T` into
`target` in the target's own dtype.  For a dtype that cannot hold it (uint8 always, int8 / int16 for large `L * T`) the
value wraps and the reference then raises from its `reshape` or counts the entries into other bins; the goldens record
that.  Here the sentinel is written into the int64 copy the mapping makes anyway (`2 * target.long()`), so the entries the
reference's mask selects — `target == ignore_index` evaluated in the target's dtype, where uint8 257 is 1 — are dropped,
which is what the reference computes whenever the sentinel fits.
"""
from __future__ import annotations

from typing import List, Optional, Union

import torch
from torch import Tensor

BINARY_LOOP_ABOVE = 50_000  # precision_recall_curve.py:204
MULTICLASS_LOOP_ABOVE = 1_000_000  # :481, on preds.numel() * num_classes = N * C * C


def normalize(preds: Tensor, normalization: str) -> Tensor:
    """The device branch of `normalize_logits_if_needed` (utilities/compute.py:223-229)."""
    condition = ((preds < 0) | (preds > 1)).any()
    return torch.where(condition, torch.sigmoid(preds) if normalization == "sigmoid" else torch.softmax(preds, dim=1), preds)


def adjust_thresholds(thresholds: Union[int, List[float], Tensor, None], device) -> Optional[Tensor]:
    """_adjust_threshold_arg (:85-93)."""
    if isinstance(thresholds, int):
        return torch.linspace(0, 1, thresholds, device=device)
    if isinstance(thresholds, list):
        return torch.tensor(thresholds, device=device)
    return thresholds


def _bincount(x: Tensor, minlength: int) -> Tensor:
    """utilities/data.py:178-210 outside deterministic mode: `torch.bincount`."""
    return torch.bincount(x, minlength=minlength) if x.numel() else torch.zeros(minlength, dtype=torch.int64, device=x.device)


# ---- binary (:164-251) -------------------------------------------------------------------------------------------------
def binary_format(preds: Tensor, target: Tensor, thresholds, ignore_index: Optional[int] = None):
    preds, target = preds.flatten(), target.flatten()
    if ignore_index is not None:
        idx = target != ignore_index
        preds, target = preds[idx], target[idx]
    return normalize(preds, "sigmoid"), target, adjust_thresholds(thresholds, preds.device)


def binary_update_vectorized(preds: Tensor, target: Tensor, thresholds: Tensor) -> Tensor:
    len_t = len(thresholds)
    preds_t = (preds.unsqueeze(-1) >= thresholds.unsqueeze(0)).long()
    unique_mapping = preds_t + 2 * target.long().unsqueeze(-1) + 4 * torch.arange(len_t, device=target.device)
    return _bincount(unique_mapping.flatten(), minlength=4 * len_t).reshape(len_t, 2, 2)


def binary_update_loop(preds: Tensor, target: Tensor, thresholds: Tensor) -> Tensor:
    len_t = len(thresholds)
    target = target == 1
    confmat = thresholds.new_empty((len_t, 2, 2), dtype=torch.int64)
    for i in range(len_t):
        preds_t = preds >= thresholds[i]
        confmat[i, 1, 1] = (target & preds_t).sum()
        confmat[i, 0, 1] = ((~target) & preds_t).sum()
        confmat[i, 1, 0] = (target & (~preds_t)).sum()
    confmat[:, 0, 0] = len(preds_t) - confmat[:, 0, 1] - confmat[:, 1, 0] - confmat[:, 1, 1]
    return confmat


def binary_update(preds: Tensor, target: Tensor, thresholds: Tensor) -> Tensor:
    if preds.numel() <= BINARY_LOOP_ABOVE:
        return binary_update_vectorized(preds, target, thresholds)
    return binary_update_loop(preds, target, thresholds)


def binary(preds: Tensor, target: Tensor, thresholds, ignore_index: Optional[int] = None) -> Tensor:
    p, t, thr = binary_format(preds, target, thresholds, ignore_index)
    return binary_update(p, t, thr)


# ---- multiclass (:430-533) ---------------------------------------------------------------------------------------------
def multiclass_format(preds: Tensor, target: Tensor, num_classes: int, thresholds, ignore_index: Optional[int] = None,
                      average: Optional[str] = None):
    preds = preds.transpose(0, 1).reshape(num_classes, -1).T
    target = target.flatten()
    if ignore_index is not None:
        idx = target != ignore_index
        preds, target = preds[idx], target[idx]
    preds = normalize(preds, "softmax")
    if average == "micro":
        preds = preds.flatten()
        target = torch.nn.functional.one_hot(target, num_classes=num_classes).flatten()
    return preds, target, adjust_thresholds(thresholds, preds.device)


def multiclass_update_vectorized(preds: Tensor, target: Tensor, num_classes: int, thresholds: Tensor) -> Tensor:
    len_t = len(thresholds)
    preds_t = (preds.unsqueeze(-1) >= thresholds.unsqueeze(0).unsqueeze(0)).long()
    target_t = torch.nn.functional.one_hot(target, num_classes=num_classes)
    unique_mapping = preds_t + 2 * target_t.long().unsqueeze(-1)
    unique_mapping += 4 * torch.arange(num_classes, device=preds.device).unsqueeze(0).unsqueeze(-1)
    unique_mapping += 4 * num_classes * torch.arange(len_t, device=preds.device)
    return _bincount(unique_mapping.flatten(), minlength=4 * num_classes * len_t).reshape(len_t, num_classes, 2, 2)


def multiclass_update_loop(preds: Tensor, target: Tensor, num_classes: int, thresholds: Tensor) -> Tensor:
    len_t = len(thresholds)
    target_t = torch.nn.functional.one_hot(target, num_classes=num_classes)
    confmat = thresholds.new_empty((len_t, num_classes, 2, 2), dtype=torch.int64)
    for i in range(len_t):
        preds_t = preds >= thresholds[i]
        confmat[i, :, 1, 1] = (target_t & preds_t).sum(dim=0)
        confmat[i, :, 0, 1] = ((~target_t) & preds_t).sum(dim=0)
        confmat[i, :, 1, 0] = (target_t & (~preds_t)).sum(dim=0)
    confmat[:, :, 0, 0] = len(preds_t) - confmat[:, :, 0, 1] - confmat[:, :, 1, 0] - confmat[:, :, 1, 1]
    return confmat


def multiclass_update(preds: Tensor, target: Tensor, num_classes: int, thresholds: Tensor,
                      average: Optional[str] = None) -> Tensor:
    if average == "micro":
        return binary_update(preds, target, thresholds)
    if preds.numel() * num_classes <= MULTICLASS_LOOP_ABOVE:
        return multiclass_update_vectorized(preds, target, num_classes, thresholds)
    return multiclass_update_loop(preds, target, num_classes, thresholds)


def multiclass(preds: Tensor, target: Tensor, num_classes: int, thresholds, ignore_index: Optional[int] = None,
               average: Optional[str] = None) -> Tensor:
    p, t, thr = multiclass_format(preds, target, num_classes, thresholds, ignore_index, average)
    return multiclass_update(p, t, num_classes, thr, average)


# ---- multilabel (:745-799) ---------------------------------------------------------------------------------------------
def multilabel(preds: Tensor, target: Tensor, num_labels: int, thresholds, ignore_index: Optional[int] = None) -> Tensor:
    preds = preds.transpose(0, 1).reshape(num_labels, -1).T
    target = target.transpose(0, 1).reshape(num_labels, -1).T
    preds = normalize(preds, "sigmoid")
    thresholds = adjust_thresholds(thresholds, preds.device)
    if ignore_index is not None:
        sentinel = -4 * num_labels * len(thresholds)
        idx = target == ignore_index  # in the target's dtype
        preds, target = preds.clone(), target.to(torch.int64, copy=True)  # the sentinel goes into an int64 copy (docstring)
        preds[idx] = sentinel
        target[idx] = sentinel
    return _multilabel_update(preds, target, num_labels, thresholds)


def _multilabel_update(preds: Tensor, target: Tensor, num_labels: int, thresholds: Tensor) -> Tensor:
    len_t = len(thresholds)
    preds_t = (preds.unsqueeze(-1) >= thresholds.unsqueeze(0).unsqueeze(0)).long()
    unique_mapping = preds_t + 2 * target.long().unsqueeze(-1)
    unique_mapping += 4 * torch.arange(num_labels, device=preds.device).unsqueeze(0).unsqueeze(-1)
    unique_mapping += 4 * num_labels * torch.arange(len_t, device=preds.device)
    unique_mapping = unique_mapping[unique_mapping >= 0]
    return _bincount(unique_mapping, minlength=4 * num_labels * len_t).reshape(len_t, num_labels, 2, 2)


# ---- the rule, for tests that pick a path --------------------------------------------------------------------------------
def compare_dtype(score_dtype: torch.dtype, threshold_dtype: torch.dtype, n: int, num_classes: int = 1,
                  multilabel: bool = False) -> torch.dtype:
    """The dtype the chain above compares `score >= threshold` in, for a formatted batch of n rows."""
    loop = not multilabel and (n > BINARY_LOOP_ABOVE if num_classes == 1 else n * num_classes * num_classes > MULTICLASS_LOOP_ABOVE)
    return score_dtype if loop else torch.promote_types(score_dtype, threshold_dtype)


# ---- inputs the goldens and the GPU suite regenerate from a seed -----------------------------------------------------------
_BITS = {torch.float16: torch.int16, torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}


def scores_near(points: Tensor, shape, dtype: torch.dtype, seed: int) -> Tensor:
    """Scores of `dtype` in [0, 1]: a quarter uniform, the rest on one of `points` (float64) rounded to `dtype` and moved by
    -2..2 units in the last place — the values on which a comparison in another dtype gives a different answer."""
    g = torch.Generator().manual_seed(seed)
    n = 1
    for s in shape:
        n *= s
    x = torch.rand(n, generator=g, dtype=torch.float64).to(dtype)
    pick = torch.randint(0, len(points), (n,), generator=g)
    near = points.to(torch.float64)[pick].to(dtype)
    step = torch.randint(-2, 3, (n,), generator=g)
    bits = near.view(_BITS[dtype]).to(torch.int64)
    moved = torch.where(bits > 0, (bits + step).clamp(min=0), bits)  # positive values only, never across zero into NaN
    near = moved.to(_BITS[dtype]).view(dtype).clamp(0, 1)
    keep = torch.rand(n, generator=g) < 0.25
    return torch.where(keep, x, near).reshape(shape)
