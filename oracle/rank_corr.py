"""Float64 numpy oracle of the rank correlations (SpearmanCorrCoef, KendallRankCorrCoef), and torch restatements of the
reference's per-row loops for the benchmark.

Conventions (the reference's, and K17's): -0 equals +0; NaN sorts after +inf and each NaN is a tie group of its own;
Kendall counts concordant / discordant pairs over the rows where neither value is NaN, while its tie terms and row count
cover the whole column.  Pair counts and tie terms are exact integers; everything after them is float64.  The inversion
count is O(n log n), so 10^7 rows take seconds.
"""
from __future__ import annotations

import math

import numpy as np


def _as_numpy(x) -> np.ndarray:
    if hasattr(x, "detach"):
        x = x.detach().cpu()
        if str(x.dtype) == "torch.bfloat16":
            x = x.float()
        x = x.numpy()
    return np.asarray(x)


def dense_ranks(x) -> tuple[np.ndarray, np.ndarray]:
    """(dense rank per element, NaN mask) of a 1-d array: equal values share a rank, each NaN gets its own after every
    number, in arrival order."""
    x = _as_numpy(x)
    if x.dtype.kind == "f":
        nan = np.isnan(x)
        v = np.where(nan, 0.0, x.astype(np.float64) + 0.0)  # + 0.0 turns -0 into +0
        order = np.lexsort((v, nan))  # stable: NaNs last, in arrival order
    else:
        nan = np.zeros(x.shape, bool)
        v = x.astype(np.int64)
        order = np.argsort(v, kind="stable")
    sv, sn = v[order], nan[order]
    head = np.ones(len(x), bool)
    if len(x) > 1:
        head[1:] = (sv[1:] != sv[:-1]) | sn[1:]
    ranks = np.empty(len(x), np.int64)
    ranks[order] = np.cumsum(head) - 1
    return ranks, nan


def average_ranks(x) -> np.ndarray:
    """1-based ranks with ties averaged (float64)."""
    dense, _ = dense_ranks(x)
    counts = np.bincount(dense)
    ends = np.cumsum(counts)
    starts = ends - counts
    return (starts[dense] + ends[dense] + 1) / 2.0


def spearman(preds, target, eps: float = 1e-6) -> np.ndarray:
    """Spearman's rho per column of ``[N]`` / ``[N, d]`` inputs, float64 (the reference's population moments and eps)."""
    p, t = _as_numpy(preds), _as_numpy(target)
    if p.ndim == 1:
        p, t = p[:, None], t[:, None]
    out = []
    for c in range(p.shape[1]):
        rx, ry = average_ranks(p[:, c]), average_ranks(t[:, c])
        dx, dy = rx - rx.mean(), ry - ry.mean()
        cov = (dx * dy).mean()
        r = cov / (math.sqrt((dx * dx).mean()) * math.sqrt((dy * dy).mean()) + eps)
        out.append(min(1.0, max(-1.0, r)))
    return np.array(out)


def count_inversions(s) -> int:
    """Number of pairs i < j with s[i] > s[j] (non-negative integers), one bit level at a time: at level b every run of
    equal higher bits is stably partitioned by bit b after counting, for each 0-bit, the 1-bits before it in its run."""
    cur = np.asarray(s, np.int64).copy()
    n = len(cur)
    if n < 2:
        return 0
    idx = np.arange(n)
    inv = 0
    for b in range(int(cur.max()).bit_length() - 1, -1, -1):
        grp = cur >> (b + 1)
        bit = (cur >> b) & 1
        head = np.ones(n, bool)
        head[1:] = grp[1:] != grp[:-1]
        start = np.maximum.accumulate(np.where(head, idx, 0))
        ones_excl = np.cumsum(bit) - bit
        before = ones_excl - ones_excl[start]
        zero = bit == 0
        inv += int(before[zero].sum())
        gid = np.cumsum(head) - 1
        zeros_in_group = np.bincount(gid, weights=zero, minlength=int(gid[-1]) + 1).astype(np.int64)
        dst = np.where(zero, idx - before, start + zeros_in_group[gid] + before)
        nxt = np.empty_like(cur)
        nxt[dst] = cur
        cur = nxt
    return inv


def _pairs(counts: np.ndarray) -> int:
    c = counts.astype(np.int64)
    return int((c * (c - 1) // 2).sum())


def kendall_stats(x, y) -> dict:
    """Exact integer statistics of one column pair: concordant / discordant pairs and the tie terms."""
    dx, nx = dense_ranks(x)
    dy, ny = dense_ranks(y)
    n = len(dx)
    valid = ~(nx | ny)
    vx, vy = dx[valid], dy[valid]
    m = len(vx)
    disc = 0
    n1 = n2 = n3 = 0
    if m:
        order = np.lexsort((vy, vx))
        disc = count_inversions(vy[order])
        n1 = _pairs(np.bincount(vx))
        n2 = _pairs(np.bincount(vy))
        n3 = _pairs(np.unique(vx * (int(vy.max()) + 1) + vy, return_counts=True)[1])
    conc = m * (m - 1) // 2 - n1 - n2 + n3 - disc
    out = {"n": n, "conc": conc, "disc": disc}
    for name, d in (("x", dx), ("y", dy)):
        # exact Python integers over the distinct tie-group sizes (few, however long the column)
        sizes, mult = np.unique(np.bincount(d), return_counts=True) if n else (np.zeros(0, np.int64), np.zeros(0, np.int64))
        tm = [(int(t), int(k)) for t, k in zip(sizes, mult)]
        out[f"ties_{name}"] = sum(k * (t * (t - 1) // 2) for t, k in tm)
        out[f"p1_{name}"] = sum(k * t * (t - 1) * (t - 2) for t, k in tm)
        out[f"p2_{name}"] = sum(k * t * (t - 1) * (2 * t + 5) for t, k in tm)
        out[f"distinct_{name}"] = int(d.max()) + 1 if n else 0
    return out


def total_pairs_tied(s: dict) -> bool:
    total = s["n"] * (s["n"] - 1) // 2
    return s["ties_x"] == total or s["ties_y"] == total


def _phi(t: float) -> float:
    return 0.5 * math.erfc(-t / math.sqrt(2.0)) if not math.isnan(t) else math.nan


def _div(a: float, b: float) -> float:
    if b == 0:
        return math.nan if a == 0 or math.isnan(a) else math.copysign(math.inf, a)
    return a / b


def kendall(preds, target, variant: str = "b", alternative=None) -> tuple[np.ndarray, np.ndarray]:
    """(tau, p-value) per column, float64; the p-value is NaN when ``alternative`` is None."""
    p, t = _as_numpy(preds), _as_numpy(target)
    if p.ndim == 1:
        p, t = p[:, None], t[:, None]
    taus, pvals = [], []
    for c in range(p.shape[1]):
        s = kendall_stats(p[:, c], t[:, c])
        n, cmd = s["n"], s["conc"] - s["disc"]
        if variant == "a":
            tau = _div(cmd, s["conc"] + s["disc"])
        elif variant == "b":
            total = n * (n - 1) // 2
            tau = _div(cmd, math.sqrt((total - s["ties_x"]) * (total - s["ties_y"])))
        else:
            mc = min(s["distinct_x"], s["distinct_y"])
            tau = _div(2.0 * cmd, (mc - 1) / mc * n * n) if mc else math.nan
        tau = tau if math.isnan(tau) else min(1.0, max(-1.0, tau))
        base = n * (n - 1) * (2 * n + 5)
        if variant == "a":
            tv = _div(3.0 * cmd, math.sqrt(base / 2))
        else:
            mm = n * (n - 1)
            den = (base - s["p2_x"] - s["p2_y"]) / 18
            den += _div(2.0 * s["ties_x"] * s["ties_y"], mm)
            den += _div(float(s["p1_x"]) * float(s["p1_y"]), 9.0 * mm * (n - 2))
            if total_pairs_tied(s):
                den = 0.0  # Var(S) is exactly 0 when every pair is tied in one variable
            tv = _div(cmd, math.sqrt(den)) if not (math.isnan(den) or den < 0) else math.nan
        pv = math.nan
        if alternative is not None:
            if alternative == "two-sided":
                tv = -abs(tv)
            elif alternative == "greater":
                tv = -tv
            pv = _phi(tv) * (2.0 if alternative == "two-sided" else 1.0)
        taus.append(tau)
        pvals.append(pv)
    return np.array(taus), np.array(pvals)


# ---- torch restatements of the reference's loops (benchmark baselines) ------------------------------------------------------
def torch_spearman_loop(preds, target, eps: float = 1e-6):
    """The reference's algorithm as torch ops on the inputs' device: argsort ranks in the input dtype, then one masked mean
    per repeated value."""
    import torch

    def rank(x):
        r = torch.empty_like(x)
        r[x.argsort()] = torch.arange(1, x.numel() + 1, dtype=x.dtype, device=x.device)
        s = x.sort().values
        change = torch.cat([torch.ones(1, dtype=torch.bool, device=x.device), s[1:] != s[:-1]])
        starts = torch.nonzero(change).flatten()
        counts = torch.diff(torch.cat([starts, torch.tensor([x.numel()], device=x.device)]))
        for v in s[starts[counts > 1]]:
            sel = x == v
            r[sel] = r[sel].mean()
        return r

    p = preds if preds.ndim == 2 else preds[:, None]
    t = target if target.ndim == 2 else target[:, None]
    rp = torch.stack([rank(c) for c in p.T]).T
    rt = torch.stack([rank(c) for c in t.T]).T
    dp, dt = rp - rp.mean(0), rt - rt.mean(0)
    out = ((dp * dt).mean(0) / ((dp * dp).mean(0).sqrt() * (dt * dt).mean(0).sqrt() + eps)).clamp(-1.0, 1.0)
    return out if preds.ndim == 2 else out[0]


def torch_kendall_pairs_loop(preds, target):
    """The reference's pair count as torch ops: sort by ``preds``, then one comparison of each row with all later rows.
    Returns (concordant, discordant) per column."""
    import torch

    p = preds if preds.ndim == 2 else preds[:, None]
    t = target if target.ndim == 2 else target[:, None]
    x, perm = p.T.sort()
    y = torch.gather(t.T, 1, perm).T
    x = x.T
    conc, disc = [], []
    for i in range(x.shape[0]):
        xl, xr, yl, yr = x[i], x[i + 1:], y[i], y[i + 1:]
        conc.append(((xl < xr) & (yl < yr)).sum(0))
        disc.append((((xl > xr) & (yl < yr)) | ((xl < xr) & (yl > yr))).sum(0))
    return torch.stack(conc).sum(0), torch.stack(disc).sum(0)
