"""Oracle for exact-mode curve evaluation (K3 / K5), restated in torch so that it runs on the same device as the kernels.
TEST INFRASTRUCTURE ONLY — see oracle/__init__.py.

Two forms:
  * the reference chain: `binary_clf_curve` (functional/classification/precision_recall_curve.py:30-82), the binary /
    multiclass / multilabel format steps with their `ignore_index` filters, and the ROC / PR / AUROC / AP computes.
    `documented_order=True` replaces the reference's argsort (`stable=False`, any order inside a run of equal scores) by the
    order the kernels fix: stable, descending, NaN first, and inside a run of NaN, of +inf or of -inf the negatives before
    the positives.  Those runs are the only ties the reference splits into one threshold per element (NaN - NaN and
    inf - inf are NaN, which `torch.where` counts as nonzero), so they are the only ties where the order shows.
  * the grouped form for sizes where a host sort is out of the question: `grouped_counts` bins (score code, label) with
    `torch.bincount` in int64; the cumulative sums are the exact fps / tps at every distinct score, and `auroc_exact` /
    `average_precision_exact` follow in int64 and float64.  It shares nothing with the kernels.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor


def is_special(preds: Tensor) -> Tensor:
    """NaN, +inf or -inf: the scores whose runs the reference splits into one threshold per element."""
    return ~torch.isfinite(preds)


def documented_argsort(preds: Tensor, positive: Tensor) -> Tensor:
    """Stable descending argsort, every NaN first whatever its sign bit (torch's CUDA sort puts float16 / bfloat16 NaNs with
    the sign bit set last); inside NaN / +inf / -inf runs the negatives before the positives."""
    second = torch.where(is_special(preds), positive.long(), torch.zeros_like(positive, dtype=torch.long))
    canon = torch.where(preds.isnan(), torch.full_like(preds, float("nan")), preds)
    o1 = torch.argsort(second, stable=True)
    o2 = torch.argsort(canon[o1], descending=True, stable=True)
    return o1[o2]


def binary_clf_curve(preds: Tensor, target: Tensor, sample_weights: Optional[Tensor] = None, pos_label: int = 1,
                     documented_order: bool = False):
    """`_binary_clf_curve` step by step; with `documented_order` the argsort of the kernels (see the module docstring)."""
    with torch.no_grad():
        if preds.ndim > target.ndim:
            preds = preds[:, 0]
        if documented_order:
            desc = documented_argsort(preds, target == pos_label)
        else:
            desc = torch.argsort(preds, descending=True)
        preds = preds[desc]
        target = target[desc]
        weight = sample_weights[desc] if sample_weights is not None else 1.0
        distinct = torch.where(preds[1:] - preds[:-1])[0]
        idx = torch.nn.functional.pad(distinct, [0, 1], value=target.size(0) - 1)
        target = (target == pos_label).to(torch.long)
        tps = torch.cumsum(target * weight, dim=0)[idx]
        if sample_weights is not None:
            fps = torch.cumsum((1 - target) * weight, dim=0)[idx]
        else:
            fps = 1 + idx - tps
        return fps, tps, preds[idx]


# ---- format steps (the `ignore_index` filters of the reference) ---------------------------------------------------------
def normalize_logits_if_needed(x: Tensor, normalization: str) -> Tensor:
    """utilities/compute.py:216-229.  The two branches differ on NaN: the CPU one normalizes unless every score is in [0, 1]
    (a NaN fails that test), the device one only when some score is outside (a NaN passes)."""
    y = x.sigmoid() if normalization == "sigmoid" else x.softmax(1)
    if x.device.type == "cpu":
        return x if bool(torch.all((x >= 0) * (x <= 1))) else y
    return torch.where((x < 0).any() | (x > 1).any(), y, x)


def binary_format(preds: Tensor, target: Tensor, ignore_index: Optional[int] = None):
    preds, target = preds.flatten(), target.flatten()
    if ignore_index is not None:
        keep = target != ignore_index
        preds, target = preds[keep], target[keep]
    return normalize_logits_if_needed(preds, "sigmoid"), target


def multiclass_format(preds: Tensor, target: Tensor, num_classes: int, ignore_index: Optional[int] = None):
    preds = preds.transpose(0, 1).reshape(num_classes, -1).T
    target = target.flatten()
    if ignore_index is not None:
        keep = target != ignore_index
        preds, target = preds[keep], target[keep]
    return normalize_logits_if_needed(preds, "softmax"), target


def multilabel_format(preds: Tensor, target: Tensor, num_labels: int):
    preds = preds.transpose(0, 1).reshape(num_labels, -1).T
    target = target.transpose(0, 1).reshape(num_labels, -1).T
    return normalize_logits_if_needed(preds, "sigmoid"), target


def multilabel_columns(preds: Tensor, target: Tensor, num_labels: int, ignore_index: Optional[int] = None):
    """The per-label (scores, targets) the reference's multilabel compute hands to the binary compute
    (precision_recall_curve.py:826-830): `target == ignore_index` compares in the target's dtype, so the value wraps."""
    out = []
    for i in range(num_labels):
        p, t = preds[:, i], target[:, i]
        if ignore_index is not None:
            keep = ~(t == ignore_index)
            p, t = p[keep], t[keep]
        out.append((p, t))
    return out


# ---- computes ---------------------------------------------------------------------------------------------------------
def binary_roc(fps: Tensor, tps: Tensor, thr: Tensor):
    """_binary_roc_compute, exact mode (roc.py:53-78)."""
    tps = torch.cat([torch.zeros(1, dtype=tps.dtype, device=tps.device), tps])
    fps = torch.cat([torch.zeros(1, dtype=fps.dtype, device=fps.device), fps])
    thr = torch.cat([torch.ones(1, dtype=thr.dtype, device=thr.device), thr])
    fpr = torch.zeros_like(fps) if fps[-1] <= 0 else fps / fps[-1]
    tpr = torch.zeros_like(tps) if tps[-1] <= 0 else tps / tps[-1]
    return fpr, tpr, thr


def binary_pr(fps: Tensor, tps: Tensor, thr: Tensor, target: Tensor):
    """_binary_precision_recall_curve_compute, exact mode (precision_recall_curve.py:270-289).  Recall is set to one when
    every target is 0, and is 0 / 0 = NaN when no target is positive but some is neither 0 nor positive."""
    precision = tps / (tps + fps)
    recall = torch.ones_like(tps) if bool((target == 0).all()) else tps / tps[-1]
    last = precision.new_ones(1), recall.new_zeros(1)
    precision = torch.cat([precision.flip(0), last[0]])
    recall = torch.cat([recall.flip(0), last[1]])
    return precision, recall, thr.flip(0).clone()


def binary_auroc(fps: Tensor, tps: Tensor, thr: Tensor) -> Tensor:
    """_binary_auroc_compute without max_fpr (auroc.py:83-107): trapz over the ROC in the counts' dtype."""
    fpr, tpr, _ = binary_roc(fps, tps, thr)
    return torch.trapz(tpr, fpr) * 1.0


def binary_average_precision(fps: Tensor, tps: Tensor, thr: Tensor, target: Tensor) -> Tensor:
    """_binary_average_precision_compute (average_precision.py:70-75)."""
    precision, recall, _ = binary_pr(fps, tps, thr, target)
    return -torch.sum((recall[1:] - recall[:-1]) * precision[:-1])


def auroc_exact(fps: Tensor, tps: Tensor) -> float:
    """sum dFP * (TP_prev + TP) / (2 P N) over the group ends in int64 (exact: at most 2 P N < 2^61), then one float64
    division — the kernel's integer accumulator, rounded the same way.  0.0 when a class is missing."""
    fps, tps = fps.to(torch.int64), tps.to(torch.int64)
    P, N = int(tps[-1]), int(fps[-1])
    if P == 0 or N == 0:
        return 0.0
    zero = fps.new_zeros(1)
    dfp = fps - torch.cat([zero, fps[:-1]])
    acc = int((dfp * (torch.cat([zero, tps[:-1]]) + tps)).sum())
    return float(acc) / (2.0 * float(P) * float(N))


def average_precision_exact(fps: Tensor, tps: Tensor) -> float:
    """sum dTP * TP / (TP + FP) / P in float64; -0.0 without positives (the reference's value for an all-negative curve)."""
    fps, tps = fps.to(torch.float64), tps.to(torch.float64)
    P = float(tps[-1])
    if P == 0:
        return -0.0
    dtp = tps - torch.cat([tps.new_zeros(1), tps[:-1]])
    return float((dtp * tps / (tps + fps)).sum()) / P


def grouped_counts(codes: Tensor, positive: Tensor, num_codes: int, chunk: int = 1 << 26):
    """Exact (fps, tps) int64 at every distinct score of a batch whose scores are a strictly decreasing function of an
    integer code in [0, num_codes): (pos, neg) per code from int64 bincounts, then cumulative sums in code order.  Codes that
    no sample holds are dropped.  Works on 10^9 samples without sorting them."""
    bins = torch.zeros(2 * num_codes, dtype=torch.int64, device=codes.device)
    for s in range(0, codes.numel(), chunk):
        c = codes[s:s + chunk].long() * 2 + positive[s:s + chunk].long()
        bins += torch.bincount(c, minlength=2 * num_codes)
    bins = bins.view(num_codes, 2)
    held = bins.sum(1) > 0
    cum = bins[held].cumsum(0)
    return cum[:, 0], cum[:, 1]
