"""Spearman's rank correlation (reference: functional/regression/spearman.py).  Ranking, tie averaging and the moments run in
the rank-correlation kernel K17 (`mb200_spearman_corrcoef`, csrc/rankcorr.cu) instead of an argsort in the input dtype and a
Python loop over the repeated values."""
from __future__ import annotations

import torch
from torch import Tensor

from metrics_b200 import _native
from metrics_b200.functional.regression.utils import _check_data_shape_to_num_outputs
from metrics_b200.utilities.checks import _check_same_shape


def _spearman_corrcoef_update(preds: Tensor, target: Tensor, num_outputs: int) -> tuple[Tensor, Tensor]:
    """Check the inputs (reference :56-74): both floating point, the same shape, ``num_outputs`` columns."""
    if not (preds.is_floating_point() and target.is_floating_point()):
        raise TypeError(
            "Expected `preds` and `target` both to be floating point tensors, but got {pred.dtype} and {target.dtype}"
        )
    _check_same_shape(preds, target)
    _check_data_shape_to_num_outputs(preds, target, num_outputs)
    return preds, target


def _spearman_corrcoef_compute(preds: Tensor, target: Tensor, eps: float = 1e-6) -> Tensor:
    """``cov(r_x, r_y) / (std(r_x) * std(r_y) + eps)`` per column with tie-averaged ranks, clamped to [-1, 1]; a scalar for
    1-d inputs.  The ranks and their sums are exact (deviation from the reference, which ranks in the input dtype)."""
    return _native.spearman_corrcoef(preds, target, torch.promote_types(preds.dtype, target.dtype), eps)


def spearman_corrcoef(preds: Tensor, target: Tensor) -> Tensor:
    """Spearman's rank correlation coefficient of ``preds`` and ``target`` (``[N]`` or ``[N, d]``), reference :111-140."""
    preds, target = _spearman_corrcoef_update(preds, target, num_outputs=1 if preds.ndim == 1 else preds.shape[-1])
    return _spearman_corrcoef_compute(preds, target)
