"""Oracle for the exact ROC / PR-curve family (numpy).  TEST INFRASTRUCTURE ONLY — see oracle/__init__.py.

Two flavours per quantity:
  * `*_ref32`: follows the reference's op chain and dtypes (float32 counts, float32 divisions, float32 trapz / sums) —
    this is what the goldens pin bit-for-bit-ish (numpy vs ATen summation order may differ by an ulp);
  * `*_exact`: integer counts + float64 — the mathematically exact value the CUDA path targets.
"""
from __future__ import annotations

from typing import Optional

import numpy as np


def sigmoid_if_logits(preds: np.ndarray) -> np.ndarray:
    """normalize_logits_if_needed(preds, "sigmoid"), device branch (utilities/compute.py:223-229):
    cond = any(x < 0) | any(x > 1) over the whole batch tensor."""
    with np.errstate(invalid="ignore"):
        cond = (preds < 0).any() or (preds > 1).any()
    if not cond:
        return preds
    x = preds.astype(np.float32)
    return (1.0 / (1.0 + np.exp(-x, dtype=np.float32))).astype(preds.dtype)


def softmax_if_logits(preds: np.ndarray) -> np.ndarray:
    """normalize_logits_if_needed(preds, "softmax") for [N, C] (utilities/compute.py:223-229)."""
    with np.errstate(invalid="ignore"):
        cond = (preds < 0).any() or (preds > 1).any()
    if not cond:
        return preds
    x = preds.astype(np.float32)
    e = np.exp(x - x.max(axis=1, keepdims=True), dtype=np.float32)
    return (e / e.sum(axis=1, keepdims=True, dtype=np.float32)).astype(preds.dtype)


def binary_clf_curve(preds: np.ndarray, target: np.ndarray, pos_label: int = 1, sample_weights: Optional[np.ndarray] = None):
    """_binary_clf_curve (functional/classification/precision_recall_curve.py:30-82).
    Returns integer fps, tps (int64) and thresholds (preds dtype), thresholds descending; with `sample_weights` (:64, :73-78)
    fps / tps are float64 weighted cumulative sums.  float64 scores are compared as float64 (no down-cast anywhere)."""
    # :60 argsort(descending=True), NaN first like torch; inside runs of NaN, +inf or -inf (which :70 splits into one threshold
    # per element) the order the kernels fix: negatives before positives
    p64 = preds.astype(np.float64)
    nan = np.isnan(p64)
    second = np.where(~np.isfinite(p64), (target == pos_label).astype(np.int64), 0)
    order = np.lexsort((second, -np.where(nan, 0.0, p64), ~nan))
    p = preds[order]
    t = (target[order] == pos_label).astype(np.int64)  # :72
    with np.errstate(invalid="ignore"):
        distinct = np.nonzero(p[1:] - p[:-1])[0]  # :70 (NaN - NaN, inf - inf: NaN, nonzero)
    idx = np.concatenate([distinct, [t.size - 1]])  # :71
    if sample_weights is not None:
        w = np.asarray(sample_weights, dtype=np.float64)[order]  # :64
        return np.cumsum((1 - t) * w)[idx], np.cumsum(t * w)[idx], p[idx]  # :73, :78
    tps = np.cumsum(t)[idx]  # :73
    fps = 1 + idx - tps  # :80
    return fps.astype(np.int64), tps.astype(np.int64), p[idx]


def binary_roc_ref32(preds, target, pos_label: int = 1):
    """_binary_roc_compute, exact mode (roc.py:53-78), float32 like the reference."""
    fps, tps, thr = binary_clf_curve(preds, target, pos_label)
    tps = np.concatenate([[0], tps]).astype(np.float32)
    fps = np.concatenate([[0], fps]).astype(np.float32)
    thr = np.concatenate([np.ones(1, thr.dtype), thr])
    fpr = np.zeros_like(fps) if fps[-1] <= 0 else fps / fps[-1]
    tpr = np.zeros_like(tps) if tps[-1] <= 0 else tps / tps[-1]
    return fpr, tpr, thr


def _trapz32(x: np.ndarray, y: np.ndarray) -> np.float32:
    """_auc_compute_without_check -> torch.trapz (utilities/compute.py:101-109) in float32."""
    dx = (x[1:] - x[:-1]).astype(np.float32)
    ys = (y[1:] + y[:-1]).astype(np.float32)
    return np.float32((dx * ys).sum(dtype=np.float32) / np.float32(2.0))


def binary_auroc_ref32(preds, target, max_fpr: Optional[float] = None, pos_label: int = 1) -> np.float32:
    """_binary_auroc_compute (auroc.py:83-107)."""
    fpr, tpr, _ = binary_roc_ref32(preds, target, pos_label)
    if max_fpr is None or max_fpr == 1 or fpr.sum() == 0 or tpr.sum() == 0:
        return _trapz32(fpr, tpr)
    max_area = np.float32(max_fpr)
    stop = int(np.searchsorted(fpr, max_area, side="right"))  # bucketize(right=True)
    weight = (max_area - fpr[stop - 1]) / (fpr[stop] - fpr[stop - 1])
    interp_tpr = tpr[stop - 1] + weight * (tpr[stop] - tpr[stop - 1])  # lerp
    tpr2 = np.concatenate([tpr[:stop], [interp_tpr]]).astype(np.float32)
    fpr2 = np.concatenate([fpr[:stop], [max_area]]).astype(np.float32)
    partial = _trapz32(fpr2, tpr2)
    min_area = np.float32(0.5) * max_area * max_area
    return np.float32(0.5 * (1 + (partial - min_area) / (max_area - min_area)))


def binary_auroc_exact(preds, target, pos_label: int = 1) -> float:
    """Exact trapezoid area in integers: sum dFP * (TP_prev + TP) / (2 P N)  (== Mann-Whitney U / (P N))."""
    fps, tps, _ = binary_clf_curve(preds, target, pos_label)
    P, N = int(tps[-1]), int(fps[-1])
    if P == 0 or N == 0:
        return 0.0
    tp_prev = np.concatenate([[0], tps[:-1]])
    fp_prev = np.concatenate([[0], fps[:-1]])
    s = int(((fps - fp_prev).astype(object) * (tps + tp_prev).astype(object)).sum())
    return s / (2 * P * N)


def binary_prc_ref32(preds, target, pos_label: int = 1, raw_target_all_zero: Optional[bool] = None):
    """_binary_precision_recall_curve_compute, exact mode (precision_recall_curve.py:275-290)."""
    fps, tps, thr = binary_clf_curve(preds, target, pos_label)
    tps32, fps32 = tps.astype(np.float32), fps.astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        precision = tps32 / (tps32 + fps32)
        recall = tps32 / tps32[-1]
    all_zero = bool((target == 0).all()) if raw_target_all_zero is None else raw_target_all_zero
    if all_zero:  # :278 looks at the raw target
        recall = np.ones_like(recall)
    precision = np.concatenate([precision[::-1], np.ones(1, np.float32)])
    recall = np.concatenate([recall[::-1], np.zeros(1, np.float32)])
    return precision, recall, thr[::-1].copy()


def binary_average_precision_ref32(preds, target, pos_label: int = 1, raw_target_all_zero=None) -> np.float32:
    """_binary_average_precision_compute (average_precision.py:70-75)."""
    precision, recall, _ = binary_prc_ref32(preds, target, pos_label, raw_target_all_zero)
    return np.float32(-((recall[1:] - recall[:-1]) * precision[:-1]).sum(dtype=np.float32))


def binary_average_precision_exact(preds, target, pos_label: int = 1) -> float:
    fps, tps, _ = binary_clf_curve(preds, target, pos_label)
    P = int(tps[-1])
    if P == 0:
        return -0.0
    tp_prev = np.concatenate([[0], tps[:-1]])
    return float((((tps - tp_prev) / P) * (tps / (tps + fps))).sum())


def multiclass_auroc_exact(preds: np.ndarray, target: np.ndarray, num_classes: int) -> np.ndarray:
    """Per-class one-vs-rest AUROC (roc.py:176-181 loop + auroc.py:193-205), exact arithmetic."""
    return np.array([binary_auroc_exact(preds[:, c], target, pos_label=c) for c in range(num_classes)])


def multiclass_average_precision_exact(preds: np.ndarray, target: np.ndarray, num_classes: int) -> np.ndarray:
    """Per-class one-vs-rest AP; NaN for classes without positives unless every target is class 0
    (precision_recall_curve.py:278 guard as reached from :565-569)."""
    all_zero = bool((target == 0).all())
    out = []
    for c in range(num_classes):
        if (target == c).sum() == 0 and not all_zero:
            out.append(float("nan"))
        else:
            out.append(binary_average_precision_exact(preds[:, c], target, pos_label=c))
    return np.array(out)


def reduce_per_class(res: np.ndarray, average: Optional[str], weights: np.ndarray) -> np.ndarray:
    """_reduce_auroc / _reduce_average_precision (auroc.py:45-70, average_precision.py:43-67)."""
    if average is None or average == "none":
        return res
    keep = ~np.isnan(res)
    if average == "macro":
        return res[keep].mean()
    w = weights[keep] / weights[keep].sum()
    return (res[keep] * w).sum()


def binned_confmat(preds: np.ndarray, target: np.ndarray, thresholds: np.ndarray, num_classes: int = 1) -> np.ndarray:
    """Multi-threshold confusion matrix (precision_recall_curve.py:211-226 binary, :488-507 multiclass):
    confmat[i, (c,) y, pred >= thr_i].  preds already normalised; binary targets outside {0,1} are not expected."""
    thr = np.asarray(thresholds, dtype=np.float32)
    if num_classes == 1:
        ge = preds.astype(np.float32)[:, None] >= thr[None, :]  # [N, T]
        out = np.zeros((thr.size, 2, 2), np.int64)
        for y in (0, 1):
            sel = target == y
            out[:, y, 1] = ge[sel].sum(0)
            out[:, y, 0] = sel.sum() - out[:, y, 1]
        return out
    out = np.zeros((thr.size, num_classes, 2, 2), np.int64)
    for c in range(num_classes):
        ge = preds[:, c].astype(np.float32)[:, None] >= thr[None, :]
        for y in (0, 1):
            sel = (target == c) == bool(y)
            out[:, c, y, 1] = ge[sel].sum(0)
            out[:, c, y, 0] = sel.sum() - out[:, c, y, 1]
    return out


# ----------------------------------------------------------------------------------------------------------------------
# multilabel: one binary problem per label (precision_recall_curve.py:745-836, roc.py:329-356, auroc.py:308-333,
# average_precision.py:284-309).  preds [N, L] already sigmoid-normalised, target [N, L].
# ----------------------------------------------------------------------------------------------------------------------
def multilabel_flatten(preds: np.ndarray, target: np.ndarray):
    """[N, L, ...] -> [N', L]  (precision_recall_curve.py:765-766: transpose(0,1).reshape(L,-1).T)."""
    L = preds.shape[1]
    return np.moveaxis(preds, 1, 0).reshape(L, -1).T, np.moveaxis(target, 1, 0).reshape(L, -1).T


def _label_column(preds: np.ndarray, target: np.ndarray, l: int, ignore_index: Optional[int]):
    p, t = preds[:, l], target[:, l]
    if ignore_index is not None:  # :826-830
        keep = t != ignore_index
        p, t = p[keep], t[keep]
    return p, t


def multilabel_auroc_exact(preds, target, ignore_index: Optional[int] = None) -> np.ndarray:
    return np.array([binary_auroc_exact(*_label_column(preds, target, l, ignore_index)) for l in range(preds.shape[1])])


def multilabel_average_precision_exact(preds, target, ignore_index: Optional[int] = None) -> np.ndarray:
    return np.array([binary_average_precision_exact(*_label_column(preds, target, l, ignore_index)) for l in range(preds.shape[1])])


def multilabel_roc_ref32(preds, target, ignore_index: Optional[int] = None):
    return [binary_roc_ref32(*_label_column(preds, target, l, ignore_index)) for l in range(preds.shape[1])]


def multilabel_prc_ref32(preds, target, ignore_index: Optional[int] = None):
    return [binary_prc_ref32(*_label_column(preds, target, l, ignore_index)) for l in range(preds.shape[1])]


def multilabel_positive_counts(target: np.ndarray) -> np.ndarray:
    """Weights of the `weighted` average: (target == 1).sum(0) (auroc.py:332)."""
    return (target == 1).sum(0).astype(np.float64)


def multilabel_micro(preds, target, ignore_index: Optional[int] = None):
    """`average="micro"`: flatten everything into one binary problem (auroc.py:319-325)."""
    p, t = preds.reshape(-1), target.reshape(-1)
    if ignore_index is not None:
        keep = t != ignore_index
        p, t = p[keep], t[keep]
    return p, t


def multilabel_binned_confmat(preds: np.ndarray, target: np.ndarray, thresholds: np.ndarray) -> np.ndarray:
    """[T, L, 2, 2] multi-threshold confusion matrix (precision_recall_curve.py:777-799); entries whose target is not
    0 / 1 (ignore_index, mapped to a negative bin by :768-774 and filtered at :797) do not count."""
    thr = np.asarray(thresholds, dtype=np.float32)
    L = preds.shape[1]
    out = np.zeros((thr.size, L, 2, 2), np.int64)
    for l in range(L):
        ge = preds[:, l].astype(np.float32)[:, None] >= thr[None, :]
        for y in (0, 1):
            sel = target[:, l] == y
            out[:, l, y, 1] = ge[sel].sum(0)
            out[:, l, y, 0] = sel.sum() - out[:, l, y, 1]
    return out
