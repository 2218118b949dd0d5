"""Oracle for the regression running-sum family (numpy, float64).  TEST INFRASTRUCTURE ONLY — see oracle/__init__.py.
Each function restates one reference `_x_update` + `_x_compute` pair (functional/regression/<file>.py)."""
from __future__ import annotations

import numpy as np

EPS = 1.17e-06


def mean_squared_error(p, t, squared=True, num_outputs=1):  # mse.py:22-58
    p, t = p.astype(np.float64), t.astype(np.float64)
    if num_outputs == 1:
        p, t = p.reshape(-1), t.reshape(-1)
    m = ((p - t) ** 2).sum(0) / t.shape[0]
    return m if squared else np.sqrt(m)


def mean_absolute_error(p, t, num_outputs=1):  # mae.py:22-60
    p, t = p.astype(np.float64), t.astype(np.float64)
    if num_outputs == 1:
        p, t = p.reshape(-1), t.reshape(-1)
    return np.abs(p - t).sum(0) / t.shape[0]


def mean_absolute_percentage_error(p, t):  # mape.py:22-65
    p, t = p.astype(np.float64), t.astype(np.float64)
    return (np.abs(p - t) / np.maximum(np.abs(t), EPS)).sum() / t.size


def symmetric_mean_absolute_percentage_error(p, t):  # symmetric_mape.py:22-66
    p, t = p.astype(np.float64), t.astype(np.float64)
    return 2 * (np.abs(p - t) / np.maximum(np.abs(t) + np.abs(p), EPS)).sum() / t.size


def weighted_mean_absolute_percentage_error(p, t):  # wmape.py:22-55
    p, t = p.astype(np.float64), t.astype(np.float64)
    return np.abs(p - t).sum() / max(np.abs(t).sum(), EPS)


def mean_squared_log_error(p, t):  # log_mse.py:22-53
    p, t = p.astype(np.float64), t.astype(np.float64)
    return ((np.log1p(p) - np.log1p(t)) ** 2).sum() / t.size


def log_cosh_error(p, t):  # log_cosh.py:32-75
    d = p.astype(np.float64) - t.astype(np.float64)
    return np.log((np.exp(d) + np.exp(-d)) / 2).sum(0) / t.shape[0]


def minkowski_distance(p, t, power):  # minkowski.py:21-60
    return (np.abs(p.astype(np.float64) - t.astype(np.float64)) ** power).sum() ** (1.0 / power)


def r2_score(p, t, multioutput="uniform_average"):  # r2.py:22-120 (adjusted = 0)
    p, t = p.astype(np.float64), t.astype(np.float64)
    n = t.shape[0]
    tss = (t * t).sum(0) - t.sum(0) * t.sum(0) / n
    rss = ((t - p) ** 2).sum(0)
    raw = 1 - rss / tss
    if multioutput == "raw_values":
        return raw
    if multioutput == "uniform_average":
        return raw.mean()
    return (tss / tss.sum() * raw).sum()


def relative_squared_error(p, t, squared=True):  # rse.py:22-90
    p, t = p.astype(np.float64), t.astype(np.float64)
    n = t.shape[0]
    rse = ((t - p) ** 2).sum(0) / ((t * t).sum(0) - t.sum(0) ** 2 / n)
    return np.mean(rse if squared else np.sqrt(rse))


def explained_variance(p, t, multioutput="uniform_average"):  # explained_variance.py:25-110
    p, t = p.astype(np.float64), t.astype(np.float64)
    n = t.shape[0]
    d = t - p
    num = (d * d).sum(0) / n - (d.sum(0) / n) ** 2
    den = (t * t).sum(0) / n - (t.sum(0) / n) ** 2
    s = 1 - num / den
    if multioutput == "raw_values":
        return s
    if multioutput == "uniform_average":
        return np.mean(s)
    return (den / den.sum() * s).sum()


def tweedie_deviance_score(p, t, power=0.0):  # tweedie_deviance.py:22-143 (domain checks omitted: valid inputs only)
    p, t = p.astype(np.float64).reshape(-1), t.astype(np.float64).reshape(-1)
    if power == 0:
        dev = (t - p) ** 2
    elif power == 1:
        with np.errstate(divide="ignore", invalid="ignore"):
            xlogy = np.where(t == 0, 0.0, t * np.log(t / p))  # _safe_xlogy, utilities/compute.py:32-44
        dev = 2 * (xlogy + p - t)
    elif power == 2:
        dev = 2 * (np.log(p / t) + t / p - 1)
    else:
        dev = 2 * (np.maximum(t, 0) ** (2 - power) / ((1 - power) * (2 - power)) - t * p ** (1 - power) / (1 - power)
                   + p ** (2 - power) / (2 - power))
    return dev.sum() / dev.size


# ---- the kernel's per-element terms (K9, csrc/regression_terms.cuh) ---------------------------------------------------
# `terms32` restates `reg_terms` operation for operation in the kernel's term precision: float32 for float32 / float16 /
# bfloat16 inputs (upcast exactly), float64 for float64 inputs.  For ops 0-4, 8 and 9 (MSE, MAE, MAPE, SMAPE, WMAPE, R2,
# EV) every operation is an IEEE-exact one (-, *, /, fabs, fmax), so these terms are bit-identical to the kernel's; the
# transcendental ops (MSLE, LogCosh, Minkowski, Tweedie) use numpy's own log / exp / pow and agree only to a few ulp.
EXACT_OPS = (0, 1, 2, 3, 4, 8, 9)
NUM_SUMS = {4: 2, 8: 3, 9: 4, 10: 4}


def terms32(op, p, t, param=0.0, eps=0.0):
    """``[K, ...]`` per-element terms of regression op ``op`` in the kernel's term precision (see above)."""
    p, t = np.asarray(p), np.asarray(t)
    f = np.float64 if np.float64 in (p.dtype, t.dtype) else np.float32
    p, t = p.astype(f), t.astype(f)
    param, eps, one, two = f(param), f(eps), f(1), f(2)
    with np.errstate(all="ignore"):
        if op == 10:  # Tweedie deviance of power `param` + the domain census
            if param == one:
                xlogy = np.where(t == 0, f(0), t * np.log(t / p))
                dev = two * (xlogy + p - t)
            elif param == two:
                dev = two * (np.log(p / t) + t / p - one)
            else:
                a, b = one - param, two - param
                dev = two * (np.power(np.fmax(t, f(0)), b) / (a * b) - t * np.power(p, a) / a + np.power(p, b) / b)
            return np.stack([dev, (p <= 0).astype(f), (t < 0).astype(f), (t == 0).astype(f)])
        d = p - t
        if op == 0:
            out = [d * d]
        elif op == 1:
            out = [np.abs(d)]
        elif op == 2:
            out = [np.abs(d) / np.fmax(np.abs(t), eps)]
        elif op == 3:
            out = [np.abs(d) / np.fmax(np.abs(t) + np.abs(p), eps)]
        elif op == 4:
            out = [np.abs(d), np.abs(t)]
        elif op == 5:
            lg = np.log1p(p) - np.log1p(t)
            out = [lg * lg]
        elif op == 6:
            out = [np.log((np.exp(d) + np.exp(-d)) / two)]
        elif op == 7:
            out = [np.power(np.abs(d), param)]
        elif op == 8:
            r = t - p
            out = [t * t, t, r * r]
        elif op == 9:
            r = t - p
            out = [r, r * r, t, t * t]
        else:
            raise ValueError(f"unknown regression op {op}")
    return np.stack(out)


def sums(op, p, t, num_outputs=1, param=0.0, eps=0.0):
    """``float64 [K, num_outputs]``: the terms of `terms32` summed in float64 over the rows of the ``[n, num_outputs]``
    row-major view — the layout `_native.regression_sums` returns.  Each output is summed along a contiguous axis, so that
    numpy's pairwise summation applies (its error grows with log n, not n)."""
    terms = terms32(op, np.asarray(p).reshape(-1, num_outputs), np.asarray(t).reshape(-1, num_outputs), param, eps)
    return np.ascontiguousarray(np.moveaxis(terms.astype(np.float64), 1, -1)).sum(-1)


def kl_divergence_rows(p, q, log_prob=False):  # kl_divergence.py:25-46 (`_kld_update`), fp64 throughout
    """Per-row KL(p || q).  Probabilities: both rows normalised to sum 1, terms with p = 0 count 0 (`_safe_xlogy`,
    utilities/compute.py:32-44); log-probabilities: sum exp(p) * (p - q)."""
    p = np.asarray(p, dtype=np.float64)
    q = np.asarray(q, dtype=np.float64)
    if log_prob:
        return (np.exp(p) * (p - q)).sum(-1)
    p = p / p.sum(-1, keepdims=True)
    q = q / q.sum(-1, keepdims=True)
    with np.errstate(divide="ignore", invalid="ignore"):
        terms = p * np.log(p / q)
    terms[p == 0] = 0.0
    return terms.sum(-1)


def kl_divergence(p, q, log_prob=False, reduction="mean"):  # kl_divergence.py:49-78
    m = kl_divergence_rows(p, q, log_prob)
    if reduction == "sum":
        return m.sum()
    if reduction == "mean":
        return m.sum() / m.shape[0]
    return m
