"""Regression functionals built on the K9 fused map-reduce kernel (reference: functional/regression/*.py).

Each `_x_update` returns the same sums as the reference's (float32 tensors, or the input dtype for float64), produced
by ONE kernel pass instead of 2-5 elementwise/reduction launches; the `_x_compute` halves follow the reference op for op.
"""
from __future__ import annotations

import math
from typing import Optional, Union

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200 import _native
from metrics_b200.utilities.checks import _check_same_shape
from metrics_b200.utilities.exceptions import TorchMetricsUserError

_EPS = 1.17e-06


def _sums(preds: Tensor, target: Tensor, op: int, num_outputs: int = 1, param: float = 0.0, eps: float = 0.0) -> Tensor:
    """The op's sums in the dtype the reference's ``preds - target`` has (the promoted dtype of the inputs)."""
    return _native.regression_sums(preds, target, op, num_outputs, param, eps).to(_native.regression_compute_dtype(preds, target))


def _dim0_sums(preds: Tensor, target: Tensor, op: int) -> list[Tensor]:
    """Each of the op's sums over dim 0 only, shaped ``preds.shape[1:]`` (the reference's ``torch.sum(..., dim=0)``): the
    kernel sees the inputs as ``[shape[0], prod(shape[1:])]``."""
    s = _sums(preds, target, op, math.prod(preds.shape[1:]))
    return [row.reshape(preds.shape[1:]) for row in s]


# ---- MSE (mse.py:22-58) ----------------------------------------------------------------------------------------------
def _mean_squared_error_update(preds: Tensor, target: Tensor, num_outputs: int) -> tuple[Tensor, int]:
    _check_same_shape(preds, target)
    if num_outputs == 1:
        return _sums(preds, target, _native.REG_MSE)[0].reshape(()), target.numel()
    return _dim0_sums(preds, target, _native.REG_MSE)[0], target.shape[0]


def _mean_squared_error_compute(sum_squared_error: Tensor, num_obs: Union[int, Tensor], squared: bool = True) -> Tensor:
    return sum_squared_error / num_obs if squared else torch.sqrt(sum_squared_error / num_obs)


def mean_squared_error(preds: Tensor, target: Tensor, squared: bool = True, num_outputs: int = 1) -> Tensor:
    sse, n = _mean_squared_error_update(preds, target, num_outputs)
    return _mean_squared_error_compute(sse, n, squared)


# ---- MAE (mae.py:22-60) ----------------------------------------------------------------------------------------------
def _mean_absolute_error_update(preds: Tensor, target: Tensor, num_outputs: int = 1) -> tuple[Tensor, int]:
    _check_same_shape(preds, target)
    if num_outputs == 1:
        return _sums(preds, target, _native.REG_MAE)[0].reshape(()), target.numel()
    return _dim0_sums(preds, target, _native.REG_MAE)[0], target.shape[0]


def _mean_absolute_error_compute(sum_abs_error: Tensor, num_obs: Union[int, Tensor]) -> Tensor:
    return sum_abs_error / num_obs


def mean_absolute_error(preds: Tensor, target: Tensor, num_outputs: int = 1) -> Tensor:
    return _mean_absolute_error_compute(*_mean_absolute_error_update(preds, target, num_outputs))


# ---- MAPE / SMAPE / WMAPE (mape.py, symmetric_mape.py, wmape.py) -------------------------------------------------------
def _mean_absolute_percentage_error_update(preds: Tensor, target: Tensor, epsilon: float = _EPS) -> tuple[Tensor, int]:
    _check_same_shape(preds, target)
    return _sums(preds, target, _native.REG_MAPE, eps=epsilon)[0, 0], target.numel()


def _mean_absolute_percentage_error_compute(sum_abs_per_error: Tensor, num_obs: Union[int, Tensor]) -> Tensor:
    return sum_abs_per_error / num_obs


def mean_absolute_percentage_error(preds: Tensor, target: Tensor) -> Tensor:
    return _mean_absolute_percentage_error_compute(*_mean_absolute_percentage_error_update(preds, target))


def _symmetric_mean_absolute_percentage_error_update(preds: Tensor, target: Tensor, epsilon: float = _EPS) -> tuple[Tensor, int]:
    _check_same_shape(preds, target)
    return 2 * _sums(preds, target, _native.REG_SMAPE, eps=epsilon)[0, 0], target.numel()


def _symmetric_mean_absolute_percentage_error_compute(sum_abs_per_error: Tensor, num_obs: Union[int, Tensor]) -> Tensor:
    return sum_abs_per_error / num_obs


def symmetric_mean_absolute_percentage_error(preds: Tensor, target: Tensor) -> Tensor:
    return _symmetric_mean_absolute_percentage_error_compute(*_symmetric_mean_absolute_percentage_error_update(preds, target))


def _weighted_mean_absolute_percentage_error_update(preds: Tensor, target: Tensor) -> tuple[Tensor, Tensor]:
    _check_same_shape(preds, target)
    s = _sums(preds, target, _native.REG_WMAPE)
    return s[0, 0], s[1, 0]


def _weighted_mean_absolute_percentage_error_compute(sum_abs_error: Tensor, sum_scale: Tensor, epsilon: float = _EPS) -> Tensor:
    return sum_abs_error / torch.clamp(sum_scale, min=epsilon)


def weighted_mean_absolute_percentage_error(preds: Tensor, target: Tensor) -> Tensor:
    return _weighted_mean_absolute_percentage_error_compute(*_weighted_mean_absolute_percentage_error_update(preds, target))


# ---- MSLE (log_mse.py:22-53) -----------------------------------------------------------------------------------------
def _mean_squared_log_error_update(preds: Tensor, target: Tensor) -> tuple[Tensor, int]:
    _check_same_shape(preds, target)
    return _sums(preds, target, _native.REG_MSLE)[0, 0], target.numel()


def _mean_squared_log_error_compute(sum_squared_log_error: Tensor, num_obs: Union[int, Tensor]) -> Tensor:
    return sum_squared_log_error / num_obs


def mean_squared_log_error(preds: Tensor, target: Tensor) -> Tensor:
    return _mean_squared_log_error_compute(*_mean_squared_log_error_update(preds, target))


# ---- LogCosh (log_cosh.py:24-75) -------------------------------------------------------------------------------------
def _check_data_shape_to_num_outputs(preds: Tensor, target: Tensor, num_outputs: int) -> None:
    if preds.ndim > 2:
        raise ValueError(f"Expected both predictions and target to be either 1- or 2-dimensional tensors, but got {target.ndim} and {preds.ndim}.")
    cond1 = num_outputs == 1 and not (preds.ndim == 1 or preds.shape[1] == 1)
    cond2 = num_outputs > 1 and (preds.ndim == 1 or num_outputs != preds.shape[1])
    if cond1 or cond2:
        raise ValueError(f"Expected argument `num_outputs` to match the second dimension of input, but got {num_outputs} and {preds.shape[1] if preds.ndim > 1 else 1}.")


def _log_cosh_error_update(preds: Tensor, target: Tensor, num_outputs: int) -> tuple[Tensor, Tensor]:
    _check_same_shape(preds, target)
    _check_data_shape_to_num_outputs(preds, target, num_outputs)
    s = _sums(preds, target, _native.REG_LOGCOSH, num_outputs)[0].squeeze()
    return s, torch.tensor(target.shape[0], device=preds.device)


def _log_cosh_error_compute(sum_log_cosh_error: Tensor, num_obs: Tensor) -> Tensor:
    return (sum_log_cosh_error / num_obs).squeeze()


def log_cosh_error(preds: Tensor, target: Tensor) -> Tensor:
    s, n = _log_cosh_error_update(preds, target, num_outputs=1 if preds.ndim == 1 else preds.shape[-1])
    return _log_cosh_error_compute(s, n)


# ---- Minkowski (minkowski.py:21-60) ----------------------------------------------------------------------------------
def _minkowski_distance_update(preds: Tensor, targets: Tensor, p: float) -> Tensor:
    _check_same_shape(preds, targets)
    if not (isinstance(p, (float, int)) and p >= 1):
        raise TorchMetricsUserError(f"Argument ``p`` must be a float or int greater than 1, but got {p}")
    return _sums(preds, targets, _native.REG_MINKOWSKI, param=float(p))[0, 0]


def _minkowski_distance_compute(distance: Tensor, p: float) -> Tensor:
    return torch.pow(distance, 1.0 / p)


def minkowski_distance(preds: Tensor, targets: Tensor, p: float) -> Tensor:
    return _minkowski_distance_compute(_minkowski_distance_update(preds, targets, p), p)


# ---- R2 / RSE (r2.py:22-120, rse.py:22-60) ---------------------------------------------------------------------------
def _r2_score_update(preds: Tensor, target: Tensor) -> tuple[Tensor, Tensor, Tensor, int]:
    _check_same_shape(preds, target)
    if preds.ndim > 2:
        raise ValueError(
            "Expected both prediction and target to be 1D or 2D tensors,"
            f" but received tensors with dimension {preds.shape}"
        )
    sum_squared_obs, sum_obs, rss = _dim0_sums(preds, target, _native.REG_R2)
    return sum_squared_obs, sum_obs, rss, target.size(0)


def _r2_score_compute(
    sum_squared_obs: Tensor, sum_obs: Tensor, rss: Tensor, num_obs: Union[int, Tensor], adjusted: int = 0,
    multioutput: str = "uniform_average",
) -> Tensor:
    if num_obs < 2:
        raise ValueError("Needs at least two samples to calculate r2 score.")
    mean_obs = sum_obs / num_obs
    tss = sum_squared_obs - sum_obs * mean_obs
    cond_rss = ~torch.isclose(rss, torch.zeros_like(rss), atol=1e-4)
    cond_tss = ~torch.isclose(tss, torch.zeros_like(tss), atol=1e-4)
    cond = cond_rss & cond_tss
    raw_scores = torch.where(cond, 1 - rss / torch.where(cond, tss, torch.ones_like(tss)), torch.ones_like(rss))
    raw_scores = torch.where(cond_rss & ~cond_tss, torch.zeros_like(raw_scores), raw_scores)
    if multioutput == "raw_values":
        r2 = raw_scores
    elif multioutput == "uniform_average":
        r2 = torch.mean(raw_scores)
    elif multioutput == "variance_weighted":
        r2 = torch.sum(tss / torch.sum(tss) * raw_scores)
    else:
        raise ValueError(
            "Argument `multioutput` must be either `raw_values`,"
            f" `uniform_average` or `variance_weighted`. Received {multioutput}."
        )
    if adjusted < 0 or not isinstance(adjusted, int):
        raise ValueError("`adjusted` parameter should be an integer larger or equal to 0.")
    if adjusted != 0:
        if adjusted > num_obs - 1:
            from metrics_b200.utilities.prints import rank_zero_warn

            rank_zero_warn("More independent regressions than data points in adjusted r2 score. Falls back to standard r2 score.", UserWarning)
        elif adjusted == num_obs - 1:
            from metrics_b200.utilities.prints import rank_zero_warn

            rank_zero_warn("Division by zero in adjusted r2 score. Falls back to standard r2 score.", UserWarning)
        else:
            return 1 - (1 - r2) * (num_obs - 1) / (num_obs - adjusted - 1)
    return r2


def r2_score(preds: Tensor, target: Tensor, adjusted: int = 0, multioutput: str = "uniform_average") -> Tensor:
    sso, so, rss, n = _r2_score_update(preds, target)
    return _r2_score_compute(sso, so, rss, n, adjusted, multioutput)


def _relative_squared_error_compute(
    sum_squared_obs: Tensor, sum_obs: Tensor, sum_squared_error: Tensor, num_obs: Union[int, Tensor], squared: bool = True
) -> Tensor:
    epsilon = torch.finfo(sum_squared_error.dtype).eps
    rse = sum_squared_error / torch.clamp(sum_squared_obs - sum_obs * sum_obs / num_obs, min=epsilon)
    if not squared:
        rse = torch.sqrt(rse)
    return torch.mean(rse)


def relative_squared_error(preds: Tensor, target: Tensor, squared: bool = True) -> Tensor:
    sso, so, rss, n = _r2_score_update(preds, target)
    return _relative_squared_error_compute(sso, so, rss, n, squared)


# ---- Explained variance (explained_variance.py:25-110) ----------------------------------------------------------------
def _explained_variance_update(preds: Tensor, target: Tensor) -> tuple[int, Tensor, Tensor, Tensor, Tensor]:
    _check_same_shape(preds, target)
    sum_error, sum_squared_error, sum_target, sum_squared_target = _dim0_sums(preds, target, _native.REG_EXPVAR)
    return preds.size(0), sum_error, sum_squared_error, sum_target, sum_squared_target


def _explained_variance_compute(
    num_obs: Union[int, Tensor], sum_error: Tensor, sum_squared_error: Tensor, sum_target: Tensor, sum_squared_target: Tensor,
    multioutput: Literal["raw_values", "uniform_average", "variance_weighted"] = "uniform_average",
) -> Tensor:
    diff_avg = sum_error / num_obs
    numerator = sum_squared_error / num_obs - (diff_avg * diff_avg)
    target_avg = sum_target / num_obs
    denominator = sum_squared_target / num_obs - (target_avg * target_avg)
    nonzero_numerator = numerator != 0
    nonzero_denominator = denominator != 0
    valid = nonzero_numerator & nonzero_denominator
    scores = torch.where(valid, 1.0 - numerator / torch.where(valid, denominator, torch.ones_like(denominator)), torch.ones_like(diff_avg))
    scores = torch.where(nonzero_numerator & ~nonzero_denominator, torch.zeros_like(scores), scores)
    if multioutput == "raw_values":
        return scores
    if multioutput == "uniform_average":
        return torch.mean(scores)
    return torch.sum(denominator / torch.sum(denominator) * scores)


def explained_variance(preds: Tensor, target: Tensor, multioutput: str = "uniform_average") -> Tensor:
    if multioutput not in ("raw_values", "uniform_average", "variance_weighted"):
        raise ValueError(f"Invalid input to argument `multioutput`. Choose one of the following: ('raw_values', 'uniform_average', 'variance_weighted')")
    return _explained_variance_compute(*_explained_variance_update(preds, target), multioutput)


# ---- Tweedie deviance (tweedie_deviance.py:22-143) -------------------------------------------------------------------
def _tweedie_power_check(power: float) -> None:
    if 0 < power < 1:
        raise ValueError(f"Deviance Score is not defined for power={power}.")


def _tweedie_deviance_score_update(preds: Tensor, targets: Tensor, power: float = 0.0) -> tuple[Tensor, Tensor]:
    """Sum of the per-element deviances and their count.  ONE kernel pass produces the sum together with the census of
    out-of-domain elements the reference collects with up to two extra `torch.any` passes (:51, :59, :65-75); the census is
    read back (one sync per update, as in the reference, whose `if torch.any(...)` syncs too) and turned into the same
    ValueErrors.  Power 0 needs no domain check and is the plain squared-error sum."""
    _check_same_shape(preds, targets)
    _tweedie_power_check(power)
    num_observations = torch.tensor(preds.numel(), device=preds.device)
    if power == 0:
        return _sums(preds, targets, _native.REG_MSE)[0, 0], num_observations
    sums = _native.regression_sums(preds, targets, _native.REG_TWEEDIE, 1, float(power))[:, 0]
    deviance, bad_preds, neg_targets, zero_targets = sums.tolist()
    if power == 1:
        if bad_preds or neg_targets:
            raise ValueError(f"For power={power}, 'preds' has to be strictly positive and 'targets' cannot be negative.")
    elif power == 2:
        if bad_preds or neg_targets or zero_targets:
            raise ValueError(f"For power={power}, both 'preds' and 'targets' have to be strictly positive.")
    elif power < 0:
        if bad_preds:
            raise ValueError(f"For power={power}, 'preds' has to be strictly positive.")
    elif 1 < power < 2:
        if bad_preds or neg_targets:
            raise ValueError(f"For power={power}, 'targets' has to be strictly positive and 'preds' cannot be negative.")
    elif bad_preds or neg_targets or zero_targets:
        raise ValueError(f"For power={power}, both 'preds' and 'targets' have to be strictly positive.")
    return sums[0].to(_native.regression_compute_dtype(preds, targets)), num_observations


def _tweedie_deviance_score_compute(sum_deviance_score: Tensor, num_observations: Tensor) -> Tensor:
    return sum_deviance_score / num_observations


def tweedie_deviance_score(preds: Tensor, targets: Tensor, power: float = 0.0) -> Tensor:
    """Mean Tweedie deviance: power 0 normal, 1 Poisson, (1, 2) compound Poisson-Gamma, 2 Gamma, 3 inverse Gaussian, < 0
    extreme stable (reference :101-143)."""
    return _tweedie_deviance_score_compute(*_tweedie_deviance_score_update(preds, targets, power))


# ---- Critical success index (csi.py:22-107) --------------------------------------------------------------------------
def _critical_success_index_update(preds: Tensor, target: Tensor, threshold: float,
                                   keep_sequence_dim: Optional[int] = None) -> tuple[Tensor, Tensor, Tensor]:
    """hits / misses / false alarms of the two fields binarised at ``threshold`` (``>=``), over everything or — with
    ``keep_sequence_dim`` — separately per index of that dimension.  After the binarisation these are the tp / fn / fp of the
    binary counting kernel (K2): ONE launch, with the kept dimension presented as its label dimension, instead of the
    reference's three masked reductions (:44-51)."""
    from metrics_b200.functional.classification import _binary_counts as _bc

    _check_same_shape(preds, target)
    if keep_sequence_dim is not None and not 0 <= keep_sequence_dim < preds.ndim:
        raise ValueError(f"Expected keep_sequence dim to be in range [0, {preds.ndim}] but got {keep_sequence_dim}")
    above_p, above_t = (preds >= threshold).long(), (target >= threshold).long()
    if preds.ndim == 1:
        keep_sequence_dim = None  # nothing left to sum over: `torch.sum(x, dim=())` reduces everything (reference :47-50)
    if keep_sequence_dim is None:
        counts = _bc.counts(above_p.reshape(-1), above_t.reshape(-1), 1, 0.5, None, False, False)[0]
    else:  # [outer, S, inner]: the kernel's `[n_outer, num_labels, inner]` layout
        kept = preds.shape[keep_sequence_dim]
        as_labels = [x.movedim(keep_sequence_dim, 0).reshape(1, kept, -1) for x in (above_p, above_t)]
        counts = _bc.counts(as_labels[0], as_labels[1], kept, 0.5, None, False, False)
    tp, fp, fn = counts[..., 0], counts[..., 1], counts[..., 3]
    return tp.int(), fn.int(), fp.int()


def _critical_success_index_compute(hits: Tensor, misses: Tensor, false_alarms: Tensor) -> Tensor:
    from metrics_b200.utilities.compute import _safe_divide

    return _safe_divide(hits, hits + misses + false_alarms)


def critical_success_index(preds: Tensor, target: Tensor, threshold: float, keep_sequence_dim: Optional[int] = None) -> Tensor:
    """hits / (hits + misses + false alarms), also known as the threat score (reference :71-107)."""
    return _critical_success_index_compute(*_critical_success_index_update(preds, target, threshold, keep_sequence_dim))
