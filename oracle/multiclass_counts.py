"""Oracle for the multiclass confusion-matrix and stat-score counts (kernels K1 / K1b, csrc/confmat.cu).  TEST INFRASTRUCTURE
ONLY — see oracle/__init__.py.

Like oracle/binary_counts.py, this is the reference's own chain of torch ops, restated device-agnostically (on a GPU it runs
on the kernel's device, as the arbiter):

  * the confusion matrix: `_multiclass_confusion_matrix_format` + `_multiclass_confusion_matrix_update`
    (functional/classification/confusion_matrix.py:297-328), through `oracle.torch_cpu_chain.multiclass_confmat_update_cpu`;
  * the stat scores: `_multiclass_stat_scores_format` + `_multiclass_stat_scores_update`
    (functional/classification/stat_scores.py:328-449): the bincount branch (macro / none / weighted), the micro branch and
    the one-hot branch (`top_k > 1` and samplewise), including the remap of an `ignore_index` outside `[0, C)`.

What it pins that a numpy restatement would have to re-derive:

  * `target != ignore_index` with a Python int: ATen casts the scalar to the TARGET's dtype first, so with uint8 targets
    257 compares as 1 and -100 as 156, with int8 targets 255 as -1, with int16 65535 as -1 (bool promotes: no wrap);
  * `argmax(dim=1)`: the first maximal index, NaN maximal, -0 == +0.

`torch.topk` does not define the order of equal scores.  Rows whose k-th and (k+1)-th scores tie, or whose top-1 ties, are
therefore counted under the rule the kernel documents (DESIGN §K1b: equal scores rank by lower column index) by
`topk_refined_lowest_index`; every other row goes through the reference's chain (`stat_scores(..., top_k=k)`).
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor

from oracle.torch_cpu_chain import multiclass_confmat_update_cpu


def confusion_matrix(preds: Tensor, target: Tensor, num_classes: int, ignore_index: Optional[int] = None) -> Tensor:
    """`[C, C]` int64 counts of one update (rows = target, columns = prediction)."""
    confmat = torch.zeros(num_classes, num_classes, dtype=torch.int64, device=preds.device)
    multiclass_confmat_update_cpu(confmat, preds, target, num_classes, ignore_index)
    return confmat


def _stat_scores_format(preds: Tensor, target: Tensor, top_k: int = 1) -> tuple[Tensor, Tensor]:
    """stat_scores.py:328-344."""
    if preds.ndim == target.ndim + 1 and top_k == 1:  # :340-341
        preds = preds.argmax(dim=1)
    preds = preds.reshape(*preds.shape[:2], -1) if top_k != 1 else preds.reshape(preds.shape[0], -1)  # :342
    target = target.reshape(target.shape[0], -1)  # :343
    return preds, target


def _select_topk(prob_tensor: Tensor, topk: int, dim: int = 1) -> Tensor:
    """utilities/data.py:116-148 (select_topk + _top_k_with_half_precision_support)."""
    out = torch.zeros_like(prob_tensor, dtype=torch.int)
    if topk == 1:
        out.scatter_(dim, prob_tensor.argmax(dim=dim, keepdim=True), 1.0)
    else:
        if prob_tensor.dtype == torch.half and not prob_tensor.is_cuda:  # :118-120
            idx = torch.argsort(prob_tensor, dim=dim, stable=True).flip(dim).narrow(dim, 0, topk)
        else:
            idx = prob_tensor.topk(k=topk, dim=dim).indices
        out.scatter_(dim, idx, 1.0)
    return out.int()


def _refine_preds_oh(preds: Tensor, preds_oh: Tensor, target: Tensor, top_k: int) -> Tensor:
    """stat_scores.py:347-368."""
    preds = preds.squeeze()
    target = target.squeeze()
    top_k_indices = torch.topk(preds, k=top_k, dim=1).indices
    top_1_indices = top_k_indices[:, 0]
    target_in_topk = torch.any(top_k_indices == target.unsqueeze(1), dim=1)
    result = torch.where(target_in_topk, target, top_1_indices)
    return torch.zeros_like(preds_oh, dtype=torch.int32).scatter_(-1, result.unsqueeze(1).unsqueeze(1), 1)


def _stat_scores_update(preds: Tensor, target: Tensor, num_classes: int, top_k: int, average: Optional[str],
                        multidim_average: str, ignore_index: Optional[int]):
    """stat_scores.py:371-449, line for line."""
    if multidim_average == "samplewise" or top_k != 1:  # :390-423
        ignore_in = 0 <= ignore_index <= num_classes - 1 if ignore_index is not None else None
        if ignore_index is not None and not ignore_in:
            preds = preds.clone()
            target = target.clone()
            idx = target == ignore_index
            target[idx] = num_classes
            idx = idx.unsqueeze(1).repeat(1, num_classes, 1) if preds.ndim > target.ndim else idx
            preds[idx] = num_classes
        if top_k > 1:
            preds_oh = torch.movedim(_select_topk(preds, topk=top_k, dim=1), 1, -1)
            preds_oh = _refine_preds_oh(preds, preds_oh, target, top_k)
        else:
            preds_oh = torch.nn.functional.one_hot(
                preds.long(), num_classes + 1 if ignore_index is not None and not ignore_in else num_classes)
        target_oh = torch.nn.functional.one_hot(
            target.long(), num_classes + 1 if ignore_index is not None and not ignore_in else num_classes)
        if ignore_index is not None:
            if 0 <= ignore_index <= num_classes - 1:
                target_oh[target == ignore_index, :] = -1
            else:
                preds_oh = preds_oh[..., :-1] if top_k == 1 else preds_oh
                target_oh = target_oh[..., :-1]
                target_oh[target == num_classes, :] = -1
        sum_dim = [0, 1] if multidim_average == "global" else [1]
        tp = ((target_oh == preds_oh) & (target_oh == 1)).sum(sum_dim)
        fn = ((target_oh != preds_oh) & (target_oh == 1)).sum(sum_dim)
        fp = ((target_oh != preds_oh) & (target_oh == 0)).sum(sum_dim)
        tn = ((target_oh == preds_oh) & (target_oh == 0)).sum(sum_dim)
    elif average == "micro":  # :424-434
        preds = preds.flatten()
        target = target.flatten()
        if ignore_index is not None:
            idx = target != ignore_index
            preds = preds[idx]
            target = target[idx]
        tp = (preds == target).sum()
        fp = (preds != target).sum()
        fn = (preds != target).sum()
        tn = num_classes * preds.numel() - (fp + fn + tp)
    else:  # :435-448
        preds = preds.flatten()
        target = target.flatten()
        if ignore_index is not None:
            idx = target != ignore_index
            preds = preds[idx]
            target = target[idx]
        unique_mapping = target.to(torch.long) * num_classes + preds.to(torch.long)
        bins = torch.bincount(unique_mapping, minlength=num_classes**2)  # utilities/data.py:206
        confmat = bins.reshape(num_classes, num_classes)
        tp = confmat.diag()
        fp = confmat.sum(0) - tp
        fn = confmat.sum(1) - tp
        tn = confmat.sum() - (fp + fn + tp)
    return tp, fp, tn, fn


def stat_scores(preds: Tensor, target: Tensor, num_classes: int, top_k: int = 1, average: Optional[str] = "macro",
                multidim_average: str = "global", ignore_index: Optional[int] = None) -> Tensor:
    """`[4, ...]` int64 `(tp, fp, tn, fn)` of one update: `[4]` (micro), `[4, C]` (global) or `[4, N, C]` (samplewise).

    `top_k > 1` goes through the chain unchanged; `stat_scores_topk` splits off the rows where `torch.topk` is free to
    order equal scores either way."""
    p, t = _stat_scores_format(preds, target, top_k)
    tp, fp, tn, fn = _stat_scores_update(p, t, num_classes, top_k, average, multidim_average, ignore_index)
    return torch.stack([tp, fp, tn, fn]).to(torch.int64)


# ----------------------------------------------------------------------------------------------------------------------
# top-k rows whose order torch.topk leaves open
# ----------------------------------------------------------------------------------------------------------------------
def order_keys(preds: Tensor) -> Tensor:
    """int64 keys in the order `torch.argmax` compares scores: NaN above everything (all NaNs equal), -0 == +0."""
    x = preds if preds.dtype == torch.float64 else preds.double()
    b = x.view(torch.int64)
    keys = torch.where(b < 0, -(b & 0x7FFFFFFFFFFFFFFF), b)
    return torch.where(torch.isnan(x), torch.full_like(keys, 0x7FFFFFFFFFFFFFFF), keys)


def topk_tie_rows(preds: Tensor, top_k: int) -> Tensor:
    """`[N]` bool: the row's top-1 score ties, or its k-th and (k+1)-th scores do."""
    s = order_keys(preds).sort(dim=1, descending=True).values
    tie = s[:, 0] == s[:, 1] if s.shape[1] > 1 else torch.zeros(s.shape[0], dtype=torch.bool, device=s.device)
    if top_k < s.shape[1]:
        tie |= s[:, top_k - 1] == s[:, top_k]
    return tie


def topk_refined_lowest_index(preds: Tensor, target: Tensor, top_k: int) -> Tensor:
    """`[N]` int64 refined labels under the lowest-index rule: the target when fewer than k columns rank before it (a higher
    score, or an equal one at a lower column), else the first maximal column.  Targets outside `[0, C)` keep the argmax."""
    keys = order_keys(preds)
    n, c = keys.shape
    col = torch.arange(c, device=keys.device)
    t = target.long()
    valid = (t >= 0) & (t < c)
    kt = keys.gather(1, t.clamp(0, c - 1).unsqueeze(1))
    rank = ((keys > kt) | ((keys == kt) & (col < t.clamp(0, c - 1).unsqueeze(1)))).sum(1)
    top1 = torch.where(keys == keys.max(1, keepdim=True).values, col, c).min(1).values
    return torch.where(valid & (rank < top_k), t, top1)


def stat_scores_topk(preds: Tensor, target: Tensor, num_classes: int, top_k: int,
                     ignore_index: Optional[int] = None) -> Tensor:
    """`[4, C]` int64 counts of a `[N, C]` / `[N]` top-k update: the chain on the rows without a tie at the top-1 or k-th
    place, the lowest-index rule on the others (see the module docstring).  The chain squeezes its inputs (stat_scores.py:
    362-363), so it needs two or more rows; a part of one row is counted under the rule, which agrees with any order there."""
    tie = topk_tie_rows(preds, top_k)
    out = torch.zeros(4, num_classes, dtype=torch.int64, device=preds.device)
    free, rule = ~tie, tie.clone()
    if int(free.sum()) == 1:
        rule |= free
        free = torch.zeros_like(free)
    if bool(free.any()):
        out += stat_scores(preds[free], target[free], num_classes, top_k, "none", "global", ignore_index)
    if bool(rule.any()):
        labels = topk_refined_lowest_index(preds[rule], target[rule], top_k)
        out += stat_scores(labels, target[rule], num_classes, 1, "none", "global", ignore_index)
    return out
