"""Exact oracle of kernel K19 (Hausdorff distance of 2-D masks), numpy only, and a torch op chain that restates the
reference's pytorch engine for the benchmark.

The oracle follows the reference (functional/segmentation/hausdorff_distance.py, utils.py:284-421) step by step: edges
are the mask pixels the connectivity-1 cross erosion removes (zero border), and every candidate distance is the
reference's float32 expression with torch's dtype rules: an int spacing entry keeps its axis term in int64, a float entry
rounds it to float32, and a sum or maximum of an int64 and a float32 term is taken in float32.  numpy would promote int64
times a Python float to float64, so every float step below is an explicit float32 operation.  The minimum over target
edges is brute force over every edge pair; pairs with more than `BRUTE_LIMIT` candidates take the nearest edge row of
each column instead (exact, see DESIGN.md K19), which tests/test_oracle_hausdorff.py checks against the brute force.
"""
from __future__ import annotations

import numpy as np

EMPTY_MAX = ("max(): Expected reduction dim to be specified for input.numel() == 0. Specify the reduction dim with the "
             "'dim' argument.")
NOT_BINARY = "Input x should be binarized"
BRUTE_LIMIT = 1 << 24


def edges(m: np.ndarray) -> np.ndarray:
    """Edge pixels of a 2-D bool mask: in the mask, with an axis neighbour outside the mask or the image."""
    p = np.pad(m.astype(bool), 1)
    inner = p[1:-1, 1:-1] & p[:-2, 1:-1] & p[2:, 1:-1] & p[1:-1, :-2] & p[1:-1, 2:]
    return p[1:-1, 1:-1] & ~inner


def _term(s, d: np.ndarray):
    """``s * d`` as torch computes a Python scalar times an int64 tensor: int64, or float32."""
    if isinstance(s, (bool, int, np.integer)):
        return np.int64(s) * d
    return np.float32(s) * d.astype(np.float32)


def _f32(x: np.ndarray) -> np.ndarray:
    return x.astype(np.float32) if x.dtype != np.float32 else x


def distance(dr: np.ndarray, dc: np.ndarray, spacing, metric: str) -> np.ndarray:
    """float32 ``f(dr, dc)`` of int64 row and column distances (utils.py:260-265)."""
    a, b = _term(spacing[0], np.asarray(dr, np.int64)), _term(spacing[1], np.asarray(dc, np.int64))
    if metric == "euclidean":
        a2, b2 = a * a, b * b
        s = a2 + b2 if a2.dtype == b2.dtype == np.int64 else _f32(a2) + _f32(b2)
        return np.sqrt(_f32(s))
    if metric == "chessboard":
        return _f32(np.maximum(a, b) if a.dtype == b.dtype == np.int64 else np.maximum(_f32(a), _f32(b)))
    return _f32(a + b if a.dtype == b.dtype == np.int64 else _f32(a) + _f32(b))


def directed(ea: np.ndarray, eb: np.ndarray, spacing, metric: str) -> np.float32:
    """max over edge pixels of ``ea`` of the min over edge pixels of ``eb`` of f; both must have edges."""
    ai, aj = np.nonzero(ea)
    bi, bj = np.nonzero(eb)
    best = np.full(ai.size, np.inf, np.float32)
    if ai.size * bi.size <= BRUTE_LIMIT:
        step = max(1, BRUTE_LIMIT // max(bi.size, 1) // 4)
        for s in range(0, ai.size, step):
            dr = np.abs(ai[s:s + step, None] - bi[None])
            dc = np.abs(aj[s:s + step, None] - bj[None])
            best[s:s + step] = distance(dr, dc, spacing, metric).min(1)
        return best.max()
    for j in np.unique(bj):  # per column, the nearest edge row gives the smallest f (f is monotone in dr)
        rows = np.sort(bi[bj == j])
        k = np.searchsorted(rows, ai)
        above = np.abs(ai - rows[np.maximum(k - 1, 0)])
        below = np.abs(rows[np.minimum(k, rows.size - 1)] - ai)
        best = np.minimum(best, distance(np.minimum(above, below), np.abs(aj - j), spacing, metric))
    return best.max()


def pair_distance(p: np.ndarray, t: np.ndarray, spacing, metric: str, is_directed: bool):
    """Hausdorff distance of one pair of 2-D masks (float32), inf when exactly one mask is empty, None when both are."""
    ep, et = edges(p), edges(t)
    if not ep.any() and not et.any():
        return None
    if not ep.any() or not et.any():
        return np.float32(np.inf)
    d = directed(ep, et, spacing, metric)
    return d if is_directed else max(d, directed(et, ep, spacing, metric))


def hausdorff(preds: np.ndarray, target: np.ndarray, num_classes: int, include_background: bool = False,
              distance_metric: str = "euclidean", spacing=None, is_directed: bool = False,
              input_format: str = "one-hot") -> np.ndarray:
    """``[N, C']`` float32 distances; raises the reference's errors in its order (label range, then per pair in row-major
    order: non-binary preds, non-binary target, both masks empty).  2-D images only."""
    spacing = [1, 1] if spacing is None else list(spacing)
    if input_format == "index":
        for x in (preds, target):
            if (x < 0).any():
                raise RuntimeError("Class values must be non-negative.")
            if (x >= num_classes).any():
                raise RuntimeError("Class values must be smaller than num_classes.")
        preds = np.stack([preds == c for c in range(num_classes)], 1)
        target = np.stack([target == c for c in range(num_classes)], 1)
    if not include_background and preds.shape[1] > 1:
        preds, target = preds[:, 1:], target[:, 1:]
    out = np.zeros(preds.shape[:2], np.float32)
    for b in range(preds.shape[0]):
        for c in range(preds.shape[1]):
            p, t = preds[b, c], target[b, c]
            for x in (p, t):
                if not np.isin(x, (0, 1)).all():
                    raise ValueError(NOT_BINARY)
            d = pair_distance(p != 0, t != 0, spacing, distance_metric, is_directed)
            if d is None:
                raise RuntimeError(EMPTY_MAX)
            out[b, c] = d
    return out


# ---- the reference's pytorch engine as a torch op chain (benchmark baseline) -------------------------------------------
def chain_pair(p, t, spacing, metric: str, is_directed: bool):
    """One pair through the reference's ops on torch tensors (any device): unfold erosion of the padded masks, then the
    dense ``[pixels, edge pixels]`` distance transform per direction, scattered with the row stride ``w``."""
    import torch
    import torch.nn.functional as F  # noqa: N812

    cross = torch.tensor([[0, 1, 0], [1, 1, 1], [0, 1, 0]], dtype=torch.int32, device=p.device).flatten()

    def edge(x):
        xp = F.pad(x[None, None].float(), [1, 1, 1, 1])
        u = F.unfold(F.pad(xp, [1, 1, 1, 1]), kernel_size=3) - cross[None, :, None]
        return ((u.min(1).values.reshape(xp.shape) + 1).byte()[0, 0] ^ xp.byte()[0, 0]).bool()

    def transform(x):
        x = x.float()
        i0, j0 = torch.where(x == 0)
        i1, j1 = torch.where(x == 1)
        dr = (i1.view(-1, 1) - i0.view(1, -1)).abs()
        dc = (j1.view(-1, 1) - j0.view(1, -1)).abs()
        s0, s1 = spacing
        if metric == "euclidean":
            d = ((s0 * dr) ** 2 + (s1 * dc) ** 2).sqrt()
        elif metric == "chessboard":
            d = torch.max(s0 * dr, s1 * dc).float()
        else:
            d = (s0 * dr + s1 * dc).float()
        z = torch.zeros_like(x).view(-1)
        z[i1 * x.shape[1] + j1] = d.min(1).values
        return z.view(x.shape)

    ep, et = edge(p), edge(t)
    if not et.any() or not ep.any():
        return torch.tensor(float("inf"), device=p.device)
    d = transform(~et)[ep].max()
    return d if is_directed else torch.max(d, transform(~ep)[et].max())
