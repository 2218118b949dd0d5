"""Oracle for the binary / multilabel `(tp, fp, tn, fn)` counts (kernel K2, csrc/binary.cu).  TEST INFRASTRUCTURE ONLY — see
oracle/__init__.py.

Unlike the numpy oracles, this one is the reference's own chain of torch ops, restated device-agnostically:
`_binary_stat_scores_format` + `_binary_stat_scores_update` (functional/classification/stat_scores.py:95-134) and the
multilabel pair (stat_scores.py:681-714).  What it pins is the arithmetic the kernel must reproduce and cannot be restated
in numpy without re-deriving ATen's rules:

  * `preds > threshold` with `threshold` a Python float: ATen casts the scalar to the score dtype before comparing
    (double -> float -> half / bfloat16), so a float16 score equal to float16(0.3) is not above 0.3;
  * the sigmoid of half-precision logits is evaluated in float32 and stored in the score dtype.

The logits vote is the device branch of `normalize_logits_if_needed` (utilities/compute.py:223-229): `((x < 0) | (x > 1))
.any()` then `torch.sigmoid`.  The CPU branch votes with `torch.all((x >= 0) * (x <= 1))`; the two differ only when a
score is NaN, so the CPU goldens hold no NaN.  On a GPU the chain runs on the kernel's device, as the arbiter.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor


def is_logits(preds: Tensor) -> bool:
    """The batch-global vote: any score outside [0, 1] (NaN is inside)."""
    return bool(((preds < 0) | (preds > 1)).any())


def stat_counts(preds: Tensor, target: Tensor, threshold: float = 0.5, ignore_index: Optional[int] = None,
                multilabel: bool = False, samplewise: bool = False, logits: Optional[bool] = None) -> Tensor:
    """`[G, 4]` int64 `(tp, fp, tn, fn)` in the kernel's group order: one group (binary, global), one per sample (binary,
    samplewise), one per label (multilabel, global) or sample-major `n * L + l` (multilabel, samplewise).

    `logits` overrides the vote (None: take it on `preds`), so that a batch too large for one evaluation can be counted in
    chunks under the vote of the whole batch; global counts of the chunks add up.
    """
    if preds.is_floating_point():
        if logits is None:
            logits = is_logits(preds)
        if logits:
            preds = torch.sigmoid(preds)
        preds = preds > float(threshold)
    if multilabel:
        preds = preds.reshape(*preds.shape[:2], -1)
        target = target.reshape(*target.shape[:2], -1)
    else:
        preds = preds.reshape(preds.shape[0], -1)
        target = target.reshape(target.shape[0], -1)
    if ignore_index is not None:
        idx = target == ignore_index
        target = target.clone()
        target[idx] = -1
    if multilabel:
        sum_dim = [0, -1] if not samplewise else [-1]
    else:
        sum_dim = [0, 1] if not samplewise else [1]
    eq, pos, neg = target == preds, target == 1, target == 0
    tp = (eq & pos).sum(sum_dim)
    fp = (~eq & neg).sum(sum_dim)
    tn = (eq & neg).sum(sum_dim)
    fn = (~eq & pos).sum(sum_dim)
    return torch.stack([tp, fp, tn, fn], -1).reshape(-1, 4).to(torch.int64)
