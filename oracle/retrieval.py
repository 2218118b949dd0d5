"""Exact oracle of the retrieval metrics (kernel K16): numpy float64 restatements of the eight per-query formulas of
src/torchmetrics/functional/retrieval/*.py with this package's tie rule (equal scores keep their input order), the
grouping by index, the empty-query actions and the aggregations of retrieval/base.py.  `torch_loop` restates the
reference's per-query loop with device-agnostic torch ops: the same-GPU baseline of benchmarks/retrieval_times.py."""
from __future__ import annotations

import numpy as np

KINDS = ("map", "mrr", "precision", "recall", "hit_rate", "fall_out", "r_precision", "ndcg")


def _rank(preds: np.ndarray) -> np.ndarray:
    """Descending score order, ties by position; NaN first (torch's descending sort), -0 == +0."""
    p = np.asarray(preds, dtype=np.float32).astype(np.float64)
    key = np.where(np.isnan(p), np.inf, p + 0.0)  # NaN ranks above every number (+inf included: stable, NaN rows first)
    nan_first = np.isnan(p)
    order = np.lexsort((np.arange(len(p)), -key, ~nan_first))
    return order


def _discount(n: int, k: int) -> np.ndarray:
    d = 1.0 / np.log2(np.arange(n, dtype=np.float64) + 2.0)
    d[k:] = 0.0
    return d


def _tie_dcg(preds: np.ndarray, target: np.ndarray, k: int) -> float:
    """sklearn's tie-averaged DCG in the reference's grouping: torch.unique(-preds) groups equal numbers; every NaN is a
    group of its own after all numbers, in input order."""
    p = np.asarray(preds, dtype=np.float32).astype(np.float64) + 0.0
    t = np.asarray(target, dtype=np.float64)
    n = len(p)
    disc = _discount(n, k)
    nums = ~np.isnan(p)
    vals = np.unique(-p[nums])
    out, pos = 0.0, 0
    for v in vals:
        m = nums & (-p == v)
        c = int(m.sum())
        out += t[m].mean() * disc[pos:pos + c].sum()
        pos += c
    for i in np.flatnonzero(~nums):
        out += t[i] * disc[pos]
        pos += 1
    return out


def query_value(kind: str, preds: np.ndarray, target: np.ndarray, top_k: int | None = None, adaptive_k: bool = False) -> float:
    """The per-query value of one metric (what the reference's functional returns), float64."""
    t = np.asarray(target, dtype=np.float64)
    n = len(t)
    ranked = t[_rank(preds)]
    if kind == "ndcg":
        k = n if top_k is None else top_k
        ideal = float((np.sort(t)[::-1] * _discount(n, k)).sum())
        return 0.0 if ideal == 0 else _tie_dcg(preds, t, k) / ideal
    if kind in ("map", "mrr"):
        k = min(top_k or n, n)
        top = ranked[:k]
        if not top.sum():
            return 0.0
        if kind == "mrr":
            return 1.0 / (np.flatnonzero(top)[0] + 1.0)
        pos = np.flatnonzero(top > 0) + 1.0
        return float(np.mean(np.arange(1, len(pos) + 1) / pos))
    if kind == "precision":
        k = n if top_k is None or (adaptive_k and top_k > n) else top_k
        return 0.0 if not t.sum() else float(ranked[:min(k, n)].sum() / k)
    k = n if top_k is None else top_k
    if kind == "recall":
        return 0.0 if not t.sum() else float(ranked[:k].sum() / t.sum())
    if kind == "hit_rate":
        return float(ranked[:k].sum() > 0)
    if kind == "fall_out":
        neg = 1 - ranked
        return 0.0 if not neg.sum() else float(neg[:k].sum() / neg.sum())
    if kind == "r_precision":
        r = int(t.sum())
        return 0.0 if not r else float(ranked[:r].sum() / r)
    raise ValueError(kind)


def groups(indexes: np.ndarray, preds: np.ndarray, target: np.ndarray):
    """``[(index, preds, target)]`` per distinct index, ascending; records keep their order within a query."""
    idx = np.asarray(indexes)
    order = np.argsort(idx, kind="stable")
    uniq, starts = np.unique(idx[order], return_index=True)
    bounds = list(starts) + [len(idx)]
    return [(uniq[i], np.asarray(preds)[order[bounds[i]:bounds[i + 1]]], np.asarray(target)[order[bounds[i]:bounds[i + 1]]])
            for i in range(len(uniq))]


def is_empty(kind: str, target: np.ndarray) -> bool:
    t = np.asarray(target, dtype=np.float64)
    return not (1 - t).sum() if kind == "fall_out" else not t.sum()


def per_query(kind: str, indexes, preds, target, top_k=None, adaptive_k=False):
    """``(values float64 [Q], empty bool [Q])`` in ascending index order."""
    vals, empty = [], []
    for _, p, t in groups(indexes, preds, target):
        vals.append(query_value(kind, p, t, top_k, adaptive_k))
        empty.append(is_empty(kind, t))
    return np.array(vals), np.array(empty, dtype=bool)


def aggregate(values: np.ndarray, aggregation: str) -> float:
    v = np.asarray(values, dtype=np.float32)
    if aggregation == "mean":
        return float(v.mean(dtype=np.float64))
    if aggregation == "median":  # torch.median: the lower of the two middle values
        return float(np.sort(v)[(len(v) - 1) // 2])
    return float(v.min() if aggregation == "min" else v.max())


def compute(kind: str, indexes, preds, target, top_k=None, adaptive_k=False, empty_target_action=None, aggregation="mean"):
    """What a metric class's ``compute()`` returns (string aggregations), float64; ``ValueError`` for ``'error'``."""
    action = empty_target_action or ("pos" if kind == "fall_out" else "neg")
    vals, empty = per_query(kind, indexes, preds, target, top_k, adaptive_k)
    vals = vals.astype(np.float32).astype(np.float64)
    if empty.any():
        if action == "error":
            raise ValueError("empty query")
        if action == "skip":
            vals = vals[~empty]
        else:
            vals = np.where(empty, 1.0 if action == "pos" else 0.0, vals)
    return aggregate(vals, aggregation) if len(vals) else 0.0


def torch_loop(kind: str, indexes, preds, target, top_k=None, adaptive_k=False):
    """The reference's compute loop restated with torch ops on any device: sort by index, group sizes to the host, one
    topk / argsort / gather / sum chain per query.  Returns the float32 per-query values (empty queries give 0)."""
    import torch

    indexes, order = torch.sort(indexes, stable=True)
    preds, target = preds[order], target[order]
    sizes = torch.unique_consecutive(indexes, return_counts=True)[1].cpu().tolist()
    out = []
    for p, t in zip(torch.split(preds, sizes), torch.split(target, sizes)):
        n = p.shape[0]
        t = t.float()
        if kind == "ndcg":
            k = n if top_k is None else top_k
            disc = 1.0 / torch.log2(torch.arange(n, device=p.device) + 2.0)
            disc[k:] = 0.0
            _, inv, counts = torch.unique(-p, return_inverse=True, return_counts=True)
            ranked = torch.zeros_like(counts, dtype=torch.float32).scatter_add_(0, inv, t) / counts
            cum = disc.cumsum(0)
            ends = counts.cumsum(0) - 1
            dsum = torch.cat([cum[ends[:1]], cum[ends].diff()])
            ideal = (disc * t.sort(descending=True).values).sum()
            out.append(torch.where(ideal == 0, torch.zeros_like(ideal), (ranked * dsum).sum() / ideal))
            continue
        ranked = t[torch.sort(p, descending=True, stable=True).indices]
        if kind in ("map", "mrr"):
            top = ranked[: min(top_k or n, n)]
            if kind == "mrr":
                nz = torch.nonzero(top).view(-1)
                out.append(1.0 / (nz[0] + 1.0) if nz.numel() else torch.zeros((), device=p.device))
            else:
                pos = torch.arange(1, top.numel() + 1, device=p.device, dtype=torch.float32)[top > 0]
                out.append((torch.arange(len(pos), device=p.device, dtype=torch.float32) + 1).div(pos).mean()
                           if pos.numel() else torch.zeros((), device=p.device))
            continue
        total = t.sum()
        if kind == "precision":
            k = n if top_k is None or (adaptive_k and top_k > n) else top_k
            out.append(ranked[:k].sum() / k if total else torch.zeros((), device=p.device))
        elif kind == "recall":
            out.append(ranked[: top_k or n].sum() / total if total else torch.zeros((), device=p.device))
        elif kind == "hit_rate":
            out.append((ranked[: top_k or n].sum() > 0).float())
        elif kind == "fall_out":
            neg = 1 - ranked
            out.append(neg[: top_k or n].sum() / neg.sum() if neg.sum() else torch.zeros((), device=p.device))
        else:
            r = int(total)
            out.append(ranked[:r].sum() / r if r else torch.zeros((), device=p.device))
    return torch.stack([torch.as_tensor(x, dtype=torch.float32, device=preds.device) for x in out])
