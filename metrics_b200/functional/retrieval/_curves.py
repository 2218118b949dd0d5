"""Retrieval AUROC and precision-recall curve of one query (reference: functional/retrieval/auroc.py and
precision_recall_curve.py).  The whole input is one query: one group sort and one launch of kernel K16e / K16f; the
argument checks run first, in the reference's order, so they raise the reference's errors at the same call."""
from typing import Optional

import numpy as np
import torch
from torch import Tensor
from torch.nn.functional import pad

from metrics_b200 import _native
from metrics_b200.utilities.checks import _check_retrieval_functional_inputs


def _check_max_fpr(max_fpr) -> None:
    """The reference's (loose) check of binary_auroc, then the range the kernel can evaluate: a float32 ``max_fpr`` of 1
    or more indexes past the ROC curve in the reference (``IndexError``); here it is a ``ValueError``, as is a negative
    one."""
    if max_fpr is not None and not isinstance(max_fpr, float) and 0 < max_fpr <= 1:
        raise ValueError(f"Arguments `max_fpr` should be a float in range (0, 1], but got: {max_fpr}")
    if max_fpr is not None and max_fpr != 1 and not 0 <= np.float32(max_fpr) < 1:
        raise ValueError(f"`max_fpr` must be 1 or lie in [0, 1) after rounding to float32, but got: {max_fpr}")


def retrieval_auroc(preds: Tensor, target: Tensor, top_k: Optional[int] = None, max_fpr: Optional[float] = None) -> Tensor:
    """Area under the ROC curve of the top ``top_k`` documents; 0 when they hold no target equal to 0 or none equal to 1
    (reference auroc.py).  Scores outside [0, 1] are read as logits (sigmoid); ``max_fpr`` gives the McClish-standardised
    partial area."""
    preds, target = _check_retrieval_functional_inputs(preds, target)
    top_k = top_k or preds.shape[-1]
    if not (isinstance(top_k, int) and top_k > 0):
        raise ValueError("`top_k` has to be a positive integer or None")
    _check_max_fpr(max_fpr)
    groups = _native.retrieval_sort(None, preds, target)
    return _native.retrieval_auroc(groups, top_k, max_fpr)[0][0]


def retrieval_precision_recall_curve(preds: Tensor, target: Tensor, max_k: Optional[int] = None,
                                     adaptive_k: bool = False) -> tuple[Tensor, Tensor, Tensor]:
    """Precision and recall of the top k documents for k = 1..``max_k``, and the k used (reference
    precision_recall_curve.py): under ``adaptive_k`` the k past the number of documents is that number."""
    preds, target = _check_retrieval_functional_inputs(preds, target)
    if not isinstance(adaptive_k, bool):
        raise ValueError("`adaptive_k` has to be a boolean")
    if max_k is None:
        max_k = preds.shape[-1]
    if not (isinstance(max_k, int) and max_k > 0):
        raise ValueError("`max_k` has to be a positive integer or None")
    n = preds.shape[-1]
    if adaptive_k and max_k > n:
        topk = pad(torch.arange(1, n + 1, device=preds.device), (0, max_k - n), "constant", float(n))
    else:
        topk = torch.arange(1, max_k + 1, device=preds.device)
    groups = _native.retrieval_sort(None, preds, target)
    precision, recall, _ = _native.retrieval_pr_curve(groups, max_k, adaptive_k)
    return precision[0], recall[0], topk
