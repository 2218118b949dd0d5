"""Exact oracle of RetrievalAUROC, RetrievalPrecisionRecallCurve and RetrievalRecallAtFixedPrecision (kernels K16e and
K16f): numpy restatements of src/torchmetrics/functional/retrieval/auroc.py (-> binary_auroc) and
precision_recall_curve.py with this package's tie rule (equal scores keep their input order, NaN first, -0 == +0) and
the CUDA branch of the sigmoid vote (NaN does not vote).  Areas are float64 of exact integer sums; curve values are fp32
divisions of exact counts, as in the reference.  `torch_loop_*` restate the reference's per-query loops with
device-agnostic torch ops: the same-GPU baseline of benchmarks/retrieval_curves_times.py."""
from __future__ import annotations

import numpy as np

from oracle.retrieval import _rank, aggregate, groups


def _sigmoid32(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, dtype=np.float32)
    with np.errstate(over="ignore"):
        return (np.float32(1.0) / (np.float32(1.0) + np.exp(-x))).astype(np.float32)


def query_auroc(preds, target, top_k: int | None = None, max_fpr: float | None = None) -> float:
    """retrieval_auroc of one query, float64 (the reference's value before its fp32 trapezoid)."""
    p = np.asarray(preds, dtype=np.float32)
    t = np.asarray(target, dtype=np.float64)
    n = len(p)
    sl = _rank(p)[: n if not top_k else min(top_k, n)]
    ps, ts = p[sl], t[sl]
    if not ((ts == 0).any() and (ts == 1).any()):
        return 0.0
    if ((ps < 0) | (ps > 1)).any():
        ps = _sigmoid32(ps)
    ps = ps.astype(np.float64)
    pos = (ts == 1).astype(np.int64)
    P = int(pos.sum())
    N = len(ps) - P
    ends = np.flatnonzero(np.append(~(ps[1:] == ps[:-1]), True))  # last record of each run of equal values; NaN alone
    tp = np.cumsum(pos)[ends]
    fp = ends + 1 - tp
    tp = np.concatenate([[0], tp]).astype(np.int64)
    fp = np.concatenate([[0], fp]).astype(np.int64)
    contrib = (fp[1:] - fp[:-1]) * (tp[1:] + tp[:-1])
    if max_fpr is None or max_fpr == 1:
        return float(contrib.sum()) / (2.0 * P * N)
    m32 = np.float32(max_fpr)
    fpr32 = fp.astype(np.float32) / np.float32(N)
    stop = int(np.searchsorted(fpr32, m32, side="right"))  # bucketize(..., right=True)
    m = float(m32)
    x0, x1 = fp[stop - 1] / N, fp[stop] / N
    y0, y1 = tp[stop - 1] / P, tp[stop] / P
    y = y0 + (m - x0) / (x1 - x0) * (y1 - y0)
    with np.errstate(invalid="ignore", divide="ignore"):
        pauc = float(contrib[: stop - 1].sum()) / (2.0 * P * N) + (m - x0) * (y0 + y) * 0.5
        min_area = 0.5 * m * m
        return float(np.float64(0.5) * (1 + (pauc - min_area) / np.float64(m - min_area)))


def query_pr_curve(preds, target, max_k: int, adaptive_k: bool = False) -> tuple[np.ndarray, np.ndarray]:
    """retrieval_precision_recall_curve of one query: float32 ``(precision [max_k], recall [max_k])``."""
    t = np.asarray(target, dtype=np.float64)
    n = len(t)
    total = t.sum()
    if not total:
        return np.zeros(max_k, np.float32), np.zeros(max_k, np.float32)
    cum = np.cumsum(t[_rank(preds)][: min(max_k, n)])
    cum = np.concatenate([cum, np.full(max_k - len(cum), cum[-1])]).astype(np.float32)
    k = np.arange(1, max_k + 1)
    d = np.minimum(k, n) if adaptive_k else k
    return cum / d.astype(np.float32), cum / np.float32(total)


def recall_at_fixed_precision(precision, recall, min_precision: float) -> tuple[float, int]:
    """The reference's max over ``(recall, k)`` of the points with ``precision >= min_precision`` (fp32 comparison)."""
    precision, recall = np.asarray(precision, np.float32), np.asarray(recall, np.float32)
    ok = np.flatnonzero(precision >= np.float32(min_precision))
    if not len(ok):
        return 0.0, len(precision)
    best = recall[ok].max()
    if best == 0:
        return 0.0, len(precision)
    return float(best), int(ok[recall[ok] == best].max()) + 1


def per_query_auroc(indexes, preds, target, top_k=None, max_fpr=None):
    """``(values float64 [Q], empty bool [Q])`` in ascending index order."""
    out = [(query_auroc(p, t, top_k, max_fpr), not np.asarray(t, np.float64).sum()) for _, p, t in groups(indexes, preds, target)]
    return np.array([v for v, _ in out]), np.array([e for _, e in out], dtype=bool)


def per_query_pr_curve(indexes, preds, target, max_k=None, adaptive_k=False):
    """``(precision [Q, max_k], recall [Q, max_k], empty bool [Q])``; ``max_k=None``: the longest query."""
    gs = groups(indexes, preds, target)
    max_k = max_k or max(len(p) for _, p, _ in gs)
    rows = [query_pr_curve(p, t, max_k, adaptive_k) for _, p, t in gs]
    empty = np.array([not np.asarray(t, np.float64).sum() for _, _, t in gs], dtype=bool)
    return np.stack([r[0] for r in rows]), np.stack([r[1] for r in rows]), empty


def _apply_action(values, empty, action):
    if empty.any():
        if action == "error":
            raise ValueError("empty query")
        if action == "skip":
            return values[~empty]
        values = values.copy()
        values[empty] = 1.0 if action == "pos" else 0.0
    return values


def compute_auroc(indexes, preds, target, top_k=None, max_fpr=None, empty_target_action="neg", aggregation="mean"):
    """RetrievalAUROC.compute() for a string aggregation, float64."""
    vals, empty = per_query_auroc(indexes, preds, target, top_k, max_fpr)
    vals = _apply_action(vals.astype(np.float32).astype(np.float64), empty, empty_target_action)
    return aggregate(vals, aggregation) if len(vals) else 0.0


def compute_pr_curve(indexes, preds, target, max_k=None, adaptive_k=False, empty_target_action="neg", aggregation="mean"):
    """RetrievalPrecisionRecallCurve.compute() for a string aggregation: float64 ``(precision, recall)`` [max_k]."""
    prec, rec, empty = per_query_pr_curve(indexes, preds, target, max_k, adaptive_k)
    prec, rec = (_apply_action(x, empty, empty_target_action) for x in (prec, rec))
    if not len(prec):
        return np.zeros(prec.shape[1]), np.zeros(rec.shape[1])
    return tuple(np.array([aggregate(x[:, j], aggregation) for j in range(x.shape[1])]) for x in (prec, rec))


def torch_loop_auroc(indexes, preds, target, top_k=None, max_fpr=None):
    """The reference's RetrievalAUROC loop restated with torch ops on any device: sort by index, group sizes to the host,
    per query a topk, the 0/1 membership test, the sigmoid vote, an argsort, cumsums and a trapezoid.  Float32 per-query
    values (empty queries give their value, as the loop computes it before the empty action)."""
    import torch

    indexes, order = torch.sort(indexes, stable=True)
    preds, target = preds[order], target[order]
    sizes = torch.unique_consecutive(indexes, return_counts=True)[1].cpu().tolist()
    out = []
    for p, t in zip(torch.split(preds, sizes), torch.split(target, sizes)):
        k = min(top_k or p.shape[0], p.shape[0])
        idx = p.topk(k, sorted=True)[1]
        ts, ps = t[idx], p[idx]
        if (0 not in ts) or (1 not in ts):
            out.append(torch.zeros((), device=p.device))
            continue
        ps = torch.where(((ps < 0) | (ps > 1)).any(), ps.sigmoid(), ps)
        ti = ts.int()
        desc = torch.argsort(ps, descending=True)
        ps, ti = ps[desc], ti[desc]
        last = torch.nn.functional.pad(torch.where(ps[1:] - ps[:-1])[0], [0, 1], value=ti.numel() - 1)
        tps = torch.cumsum(ti == 1, 0)[last]
        fps = 1 + last - tps
        tps, fps = (torch.cat([torch.zeros(1, dtype=x.dtype, device=x.device), x]) for x in (tps, fps))
        fpr, tpr = fps / fps[-1], tps / tps[-1]
        if max_fpr is None or max_fpr == 1:
            out.append(torch.trapz(tpr, fpr))
            continue
        m = torch.tensor(max_fpr, device=p.device)
        stop = torch.bucketize(m, fpr, out_int32=True, right=True)
        w = (m - fpr[stop - 1]) / (fpr[stop] - fpr[stop - 1])
        tpr = torch.cat([tpr[:stop], torch.lerp(tpr[stop - 1], tpr[stop], w).view(1)])
        fpr = torch.cat([fpr[:stop], m.view(1)])
        min_area = 0.5 * m**2
        out.append(0.5 * (1 + (torch.trapz(tpr, fpr) - min_area) / (m - min_area)))
    return torch.stack([x.float() for x in out])


def torch_loop_pr_curve(indexes, preds, target, max_k=None, adaptive_k=False):
    """The reference's RetrievalPrecisionRecallCurve loop restated with torch ops: per query a topk, a padded cumsum
    and two divisions, stacked to ``[Q, max_k]`` float32 (empty queries: zero rows)."""
    import torch

    indexes, order = torch.sort(indexes, stable=True)
    preds, target = preds[order], target[order]
    sizes = torch.unique_consecutive(indexes, return_counts=True)[1].cpu().tolist()
    max_k = max_k or max(sizes)
    precisions, recalls = [], []
    for p, t in zip(torch.split(preds, sizes), torch.split(target, sizes)):
        n = p.shape[0]
        if not t.sum():
            precisions.append(torch.zeros(max_k, device=p.device))
            recalls.append(torch.zeros(max_k, device=p.device))
            continue
        if adaptive_k and max_k > n:
            topk = torch.nn.functional.pad(torch.arange(1, n + 1, device=p.device), (0, max_k - n), "constant", float(n))
        else:
            topk = torch.arange(1, max_k + 1, device=p.device)
        rel = t[p.topk(min(max_k, n))[1]].float()
        rel = torch.cumsum(torch.nn.functional.pad(rel, (0, max(0, max_k - len(rel))), "constant", 0.0), 0)
        recalls.append(rel / t.sum())
        precisions.append(rel / topk)
    return torch.stack(precisions), torch.stack(recalls)
