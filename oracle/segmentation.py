"""Segmentation overlap-count oracles.  TEST/BENCH INFRASTRUCTURE.

`counts` restates what MeanIoU / DiceScore / GeneralizedDiceScore reduce an update to — per sample and class the sums over
every spatial position of the elementwise product, of preds and of target — in numpy: int64 (with its wrap) for integer
inputs, float64 sums of values rounded to the input dtype for float inputs.  `mean_iou_scores`, `dice_scores` and
`generalized_dice_scores` restate the three per-batch epilogues in float64.

The `*_chain` functions are the reference's op sequence on torch tensors of any device: class indices expanded with
`one_hot(...).movedim(-1, 1)`, the background column sliced off, then `&` or `*` and three `sum`s over the spatial axes,
followed by each metric's epilogue.  On CPU they reproduce the reference's states; on CUDA tensors they are what the
reference executes on the GPU, the yardstick the benchmark times kernel K15 against.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch
from torch import Tensor


# ---- numpy ------------------------------------------------------------------------------------------------------------
def counts(preds: np.ndarray, target: np.ndarray, num_classes: int, include_background: bool, index: bool,
           product: str = "mul") -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(intersection, pred_sum, target_sum), each [N, C'].  Index inputs: int64 labels [N, ...], labels outside
    [0, num_classes) counted nowhere.  One-hot inputs: [N, C, ...] of one dtype, ``product`` "and" or "mul" evaluated in that
    dtype."""
    if index:
        n = preds.shape[0]
        p = preds.reshape(n, -1)
        t = target.reshape(n, -1)
        inter = np.zeros((n, num_classes), np.int64)
        psum = np.zeros((n, num_classes), np.int64)
        tsum = np.zeros((n, num_classes), np.int64)
        for i in range(n):
            pv = p[i][(p[i] >= 0) & (p[i] < num_classes)]
            tv = t[i][(t[i] >= 0) & (t[i] < num_classes)]
            hit = p[i][(p[i] == t[i]) & (p[i] >= 0) & (p[i] < num_classes)]
            psum[i] = np.bincount(pv, minlength=num_classes)
            tsum[i] = np.bincount(tv, minlength=num_classes)
            inter[i] = np.bincount(hit, minlength=num_classes)
    else:
        n, c = preds.shape[:2]
        p = preds.reshape(n, c, -1)
        t = target.reshape(n, c, -1)
        with np.errstate(over="ignore"):
            if p.dtype == np.bool_:
                prod = p & t
            elif product == "and":
                prod = np.bitwise_and(p, t)
            else:
                prod = np.multiply(p, t, dtype=p.dtype)
        acc = np.float64 if np.issubdtype(p.dtype, np.floating) else np.int64
        inter, psum, tsum = (x.astype(acc).sum(axis=2, dtype=acc) for x in (prod, p, t))
    if not include_background and inter.shape[1] > 1:
        inter, psum, tsum = inter[:, 1:], psum[:, 1:], tsum[:, 1:]
    return inter, psum, tsum


def _divide(num: np.ndarray, den: np.ndarray, zero: float) -> np.ndarray:
    num, den = np.asarray(num, np.float64), np.asarray(den, np.float64)
    out = np.full(np.broadcast(num, den).shape, zero)
    np.divide(num, den, out=out, where=den != 0)
    return out


def mean_iou_scores(inter, psum, tsum, per_class: bool) -> np.ndarray:
    """Per-sample IoU [N, C'] (per_class) or its class mean [N]."""
    val = _divide(inter, tsum + psum - inter, 0.0)
    return val if per_class else val.mean(axis=1)


def dice_scores(numerator, denominator, support, average: Optional[str]) -> np.ndarray:
    """`_dice_score_compute` in float64 on the concatenated states."""
    numerator, denominator = np.asarray(numerator, np.float64), np.asarray(denominator, np.float64)
    if average == "micro":
        numerator, denominator = numerator.sum(-1), denominator.sum(-1)
    dice = _divide(numerator, denominator, 1.0)
    if average == "macro":
        dice = dice.mean(-1)
    elif average == "weighted":
        support = np.asarray(support, np.float64)
        dice = (dice * _divide(support, support.sum(-1, keepdims=True), 1.0)).sum(-1)
    return dice


def generalized_dice_scores(inter, psum, tsum, weight_type: str, per_class: bool) -> np.ndarray:
    """Per-sample generalized dice score; an infinite weight (class absent from a sample's target) takes the maximum finite
    weight of class ``i // N`` for flat index ``i = n * C' + c``, zero if that class has none."""
    tsum = np.asarray(tsum, np.float64)
    with np.errstate(divide="ignore"):
        w = {"simple": 1.0 / tsum, "square": 1.0 / tsum**2, "linear": np.ones_like(tsum)}[weight_type]
    n = w.shape[0]
    flat = w.reshape(-1).copy()
    absent = np.isinf(flat)
    flat[absent] = 0.0
    class_max = flat.reshape(w.shape).max(axis=0)
    flat[absent] = class_max[np.flatnonzero(absent) // n]
    w = flat.reshape(w.shape)
    num = 2.0 * np.asarray(inter, np.float64) * w
    den = (tsum + np.asarray(psum, np.float64)) * w
    if not per_class:
        num, den = num.sum(1), den.sum(1)
    return _divide(num, den, 0.0)


# ---- the reference's op sequence on torch tensors -------------------------------------------------------------------------
def counts_chain(preds: Tensor, target: Tensor, num_classes: int, include_background: bool, index: bool,
                 product: str) -> tuple[Tensor, Tensor, Tensor]:
    if index:
        preds = torch.nn.functional.one_hot(preds, num_classes=num_classes).movedim(-1, 1)
        target = torch.nn.functional.one_hot(target, num_classes=num_classes).movedim(-1, 1)
    if not include_background:
        if preds.shape[1] > 1:
            preds = preds[:, 1:]
        if target.shape[1] > 1:
            target = target[:, 1:]
    axes = list(range(2, preds.ndim))
    both = preds & target if product == "and" else preds * target
    return both.sum(dim=axes), preds.sum(dim=axes), target.sum(dim=axes)


def _safe_divide_chain(num: Tensor, den: Tensor, zero: float = 0.0) -> Tensor:
    num = num if num.is_floating_point() else num.float()
    den = den if den.is_floating_point() else den.float()
    return torch.where(den != 0, num / den, torch.tensor(zero, dtype=num.dtype, device=num.device))


def mean_iou_chain(preds, target, num_classes, include_background, per_class, index) -> Tensor:
    """`mean_iou(...)`: per-sample IoU (per class) or its class mean."""
    inter, psum, tsum = counts_chain(preds, target, num_classes, include_background, index, "and")
    val = _safe_divide_chain(inter, tsum + psum - inter)
    return val if per_class else torch.mean(val, 1)


def dice_update_chain(preds, target, num_classes, include_background, index) -> tuple[Tensor, Tensor, Tensor]:
    """The three per-batch `cat` entries of DiceScore."""
    inter, psum, tsum = counts_chain(preds, target, num_classes, include_background, index, "mul")
    return 2 * inter, psum + tsum, tsum


def dice_compute_chain(numerator, denominator, average, support=None) -> Tensor:
    if average == "micro":
        numerator, denominator = torch.sum(numerator, dim=-1), torch.sum(denominator, dim=-1)
    dice = _safe_divide_chain(numerator, denominator, 1.0)
    if average == "macro":
        dice = torch.mean(dice, dim=-1)
    elif average == "weighted" and support is not None:
        dice = torch.sum(dice * _safe_divide_chain(support, torch.sum(support, dim=-1, keepdim=True), 1.0), dim=-1)
    return dice


def generalized_dice_chain(preds, target, num_classes, include_background, weight_type, per_class, index) -> Tensor:
    """`generalized_dice_score(...)`: per-sample scores."""
    inter, psum, tsum = counts_chain(preds, target, num_classes, include_background, index, "mul")
    if weight_type == "simple":
        w = 1.0 / tsum
    elif weight_type == "square":
        w = 1.0 / (tsum**2)
    else:
        w = torch.ones_like(tsum)
    flat = w.flatten()  # a view: zeroing the infinities here changes `w` before its maxima are taken
    absent = torch.isinf(flat)
    flat[absent] = 0
    flat[absent] = torch.max(w, 0).values.repeat(w.shape[0], 1).T.flatten()[absent]
    w = flat.reshape(w.shape)
    num, den = 2.0 * inter * w, (tsum + psum) * w
    if not per_class:
        num, den = torch.sum(num, 1), torch.sum(den, 1)
    return _safe_divide_chain(num, den)
