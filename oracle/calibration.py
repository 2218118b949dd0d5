"""Calibration error oracles.  TEST/BENCH INFRASTRUCTURE.

`ce_compute` restates the reference's `_ce_compute` (functional/classification/calibration_error.py:30-113) in float64
numpy: exact counts, float64 sums and divisions, so it is the answer the reference would give without its state-dtype
accumulation.  The `*_chain` functions are the reference's op chain on torch tensors (any device, built on the format and
normalisation chains of oracle/torch_cpu_chain.py): on CUDA tensors they are what the reference would execute on the GPU,
the yardstick of kernel K14a's bits there.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch
from torch import Tensor

from oracle.torch_cpu_chain import _multiclass_format_chain, normalize_logits_if_needed_chain


def bin_sums(confidences: np.ndarray, accuracies: np.ndarray, boundaries: np.ndarray):
    """Per slot of ``bucketize(conf, boundaries, right=True) - 1`` (``len(boundaries)`` slots; NaN and x >= the last
    boundary land in the last slot): int64 counts and float64 sums of the confidences and of the accuracies."""
    conf = np.asarray(confidences, dtype=np.float64).ravel()
    acc = np.asarray(accuracies, dtype=np.float64).ravel()
    b = np.asarray(boundaries, dtype=np.float64)
    idx = np.searchsorted(b, conf, side="right") - 1  # numpy orders NaN last, like bucketize's `!(b > x)` search
    idx[np.isnan(conf)] = len(b) - 1
    count = np.bincount(idx, minlength=len(b)).astype(np.int64)
    sum_conf = np.bincount(idx, weights=conf, minlength=len(b))
    sum_acc = np.bincount(idx, weights=acc, minlength=len(b))
    return count, sum_conf, sum_acc


def ce_compute(confidences: np.ndarray, accuracies: np.ndarray, boundaries: np.ndarray, norm: str = "l1",
               debias: bool = False) -> float:
    """`_ce_compute` in float64 (reference :64-113); ``boundaries`` as the reference builds them (``torch.linspace(0, 1,
    n_bins + 1, dtype=state dtype)``, widened to float64) so that bin membership is the reference's."""
    count, sum_conf, sum_acc = bin_sums(confidences, accuracies, boundaries)
    with np.errstate(divide="ignore", invalid="ignore"):
        conf_bin = np.nan_to_num(sum_conf / count)
        acc_bin = np.nan_to_num(sum_acc / count)
        prop_bin = count / count.sum()
    if norm == "l1":
        return float(np.sum(np.abs(acc_bin - conf_bin) * prop_bin))
    if norm == "max":
        return float(np.max(np.abs(acc_bin - conf_bin)))
    ce = np.sum((acc_bin - conf_bin) ** 2 * prop_bin)
    if debias:
        with np.errstate(divide="ignore", invalid="ignore"):
            ce += np.sum(np.nan_to_num((acc_bin * (acc_bin - 1) * prop_bin) / (prop_bin * np.asarray(accuracies).size - 1)))
    return float(np.sqrt(ce)) if ce > 0 else 0.0


# ----------------------------------------------------------------------------------------------------------------------
# the reference's op chain on torch tensors
# ----------------------------------------------------------------------------------------------------------------------
def multiclass_calibration_update_chain(preds: Tensor, target: Tensor, num_classes: int, ignore_index: Optional[int] = None):
    """`_multiclass_confusion_matrix_format(convert_to_labels=False)` + `_multiclass_calibration_error_update`
    (calibration_error.py:239-246): rows, ignore drop, normalize_logits_if_needed(softmax), max(dim=1), eq, float."""
    preds, target = _multiclass_format_chain(preds, target, num_classes, ignore_index)
    confidences, predictions = preds.max(dim=1)
    return confidences.float(), predictions.eq(target).float()


def binary_calibration_update_chain(preds: Tensor, target: Tensor, ignore_index: Optional[int] = None):
    """`_binary_confusion_matrix_format(threshold=0, convert_to_labels=False)` + `_binary_calibration_error_update`."""
    preds, target = preds.flatten(), target.flatten()
    if ignore_index is not None:
        keep = target != ignore_index
        preds, target = preds[keep], target[keep]
    return normalize_logits_if_needed_chain(preds, "sigmoid"), target


def ce_compute_chain(confidences: Tensor, accuracies: Tensor, n_bins: int, norm: str = "l1") -> Tensor:
    """`_binning_bucketize` + `_ce_compute` (calibration_error.py:30-113): scatter_add_ in the state dtype."""
    boundaries = torch.linspace(0, 1, n_bins + 1, dtype=confidences.dtype, device=confidences.device)
    accuracies = accuracies.to(dtype=confidences.dtype)
    acc_bin = torch.zeros(len(boundaries), device=confidences.device, dtype=confidences.dtype)
    conf_bin = torch.zeros(len(boundaries), device=confidences.device, dtype=confidences.dtype)
    count_bin = torch.zeros(len(boundaries), device=confidences.device, dtype=confidences.dtype)
    indices = torch.bucketize(confidences, boundaries, right=True) - 1
    count_bin.scatter_add_(dim=0, index=indices, src=torch.ones_like(confidences))
    conf_bin.scatter_add_(dim=0, index=indices, src=confidences)
    conf_bin = torch.nan_to_num(conf_bin / count_bin)
    acc_bin.scatter_add_(dim=0, index=indices, src=accuracies)
    acc_bin = torch.nan_to_num(acc_bin / count_bin)
    prop_bin = count_bin / count_bin.sum()
    if norm == "l1":
        return torch.sum(torch.abs(acc_bin - conf_bin) * prop_bin)
    if norm == "max":
        return torch.max(torch.abs(acc_bin - conf_bin))
    ce = torch.sum(torch.pow(acc_bin - conf_bin, 2) * prop_bin)
    return torch.sqrt(ce) if ce > 0 else torch.tensor(0)
