"""Generate tests/golden/binary_counts.npz from the UNMODIFIED reference (TorchMetrics under /root/reference), CPU tensors.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_binary_counts.py

Same import set-up as make_golden.py.  The cases pin the threshold comparison behind the binary and multilabel stat scores:
probabilities and logits in float32, float16, bfloat16 and float64, with scores placed ON the threshold rounded to the
score dtype and on its representable neighbours (for logits: on the logits around the sigmoid's crossing), at thresholds
that are not representable in half precision.  Every input set is counted by the reference's `binary_stat_scores` /
`multilabel_stat_scores` for global and samplewise counts and `ignore_index` in {None, -1, 0}; the inputs hold no NaN (the
reference's CPU and device logits votes differ only there).  tests/test_oracle_binary_counts.py replays them through
oracle/binary_counts.py.
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "_standins"))
sys.path.insert(0, "/root/reference/src")

from torchmetrics.functional.classification import binary_stat_scores, multilabel_stat_scores  # noqa: E402

DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2, torch.float64: 3}
THRESHOLDS = [0.5, 0.3, 0.1, 1 / 3, 0.7, 0.9, 0.999, 0.9999, 1e-4, 0.0, 1.0,
              # ATen rounds the scalar to float32 first, then to half precision: these two land on the other side of
              # a half-precision midpoint than one direct rounding would
              0.5 + 2**-12 + 2**-40, 0.5 + 2**-9 + 2**-40]
F16_SUBNORMAL_THRESHOLDS = [2e-6, 6e-6, 1.2e-5, 3e-5, 6e-5]
IGNORE = [None, -1, 0]
N, W, L = 4, 24, 3  # binary inputs [N, W]; multilabel [N, L, W // L]


def np_of(t: torch.Tensor) -> np.ndarray:
    """float16 / bfloat16 are stored widened to float32 (exact); the dtype code says what to narrow them back to."""
    return t.float().numpy() if t.dtype in (torch.float16, torch.bfloat16) else t.numpy()


def neighbours(x: float, dtype, k: int) -> torch.Tensor:
    """x rounded to `dtype` and its k representable neighbours on each side."""
    c = torch.tensor(x, dtype=torch.float64).to(dtype)
    if dtype in (torch.float16, torch.bfloat16):  # (no nextafter for these: walk the sorted finite values instead)
        every = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(dtype)
        every = every[torch.isfinite(every)].float().unique()
        i = int(torch.searchsorted(every, c.float()))
        return every[max(0, i - k): i + k + 1].to(dtype)
    out = [c]
    lo = hi = c
    for _ in range(k):
        lo = torch.nextafter(lo, torch.tensor(-math.inf, dtype=dtype))
        hi = torch.nextafter(hi, torch.tensor(math.inf, dtype=dtype))
        out += [lo, hi]
    return torch.stack(out)


def scores(kind: str, dtype, thr: float, g: torch.Generator) -> torch.Tensor:
    n = N * W
    if kind == "probs":
        near = neighbours(thr, dtype, 8).clamp(0, 1)
        bulk = torch.rand(n, generator=g, dtype=torch.float64).to(dtype)
    else:
        if 0.0 < thr < 1.0:
            c = math.log(thr / (1 - thr))
            near = torch.cat([neighbours(c, dtype, 12),
                              # a coarse window, so that the sigmoid of several of them rounds onto T(thr)
                              (c + torch.linspace(-0.05, 0.05, 41, dtype=torch.float64) * (1 + abs(c))).to(dtype)])
        else:
            near = torch.tensor([-100.0, -30.0, -20.0, 20.0, 30.0, 100.0], dtype=torch.float64).to(dtype)
        bulk = (torch.randn(n, generator=g, dtype=torch.float64) * 6).to(dtype)
        bulk[0] = 2.0  # the batch is logits whatever the crossing window holds
    idx = torch.randperm(n, generator=g)[: near.numel()]
    bulk[idx] = near.to(dtype)
    return bulk


def counts_of(stats: torch.Tensor) -> np.ndarray:
    return stats[..., :4].reshape(-1, 4).to(torch.int64).numpy()


def binary_counts_golden() -> dict:
    g = torch.Generator().manual_seed(2024)
    out = {}
    case = 0
    for dtype, code in DTYPE_CODE.items():
        thresholds = THRESHOLDS + (F16_SUBNORMAL_THRESHOLDS if dtype == torch.float16 else [])
        for thr in thresholds:
            for kind in ("probs", "logits"):
                for multilabel in (False, True):
                    key = f"set{case}"
                    p = scores(kind, dtype, thr, g)
                    t = torch.randint(0, 2, (N * W,), generator=g)
                    t_ign = t.clone()
                    t_ign[torch.randperm(N * W, generator=g)[: N * W // 8]] = -1
                    shape = (N, L, W // L) if multilabel else (N, W)
                    p, t, t_ign = p.reshape(shape), t.reshape(shape), t_ign.reshape(shape)
                    out[f"{key}/preds"] = np_of(p)
                    out[f"{key}/target"], out[f"{key}/target_ign"] = t.to(torch.int8).numpy(), t_ign.to(torch.int8).numpy()
                    out[f"{key}/meta"] = np.array([code, int(kind == "logits"), int(multilabel)])
                    out[f"{key}/threshold"] = np.array(thr, dtype=np.float64)
                    for ign in IGNORE:
                        tt = t_ign if ign == -1 else t
                        for mda in ("global", "samplewise"):
                            if multilabel:
                                s = multilabel_stat_scores(p, tt, L, threshold=thr, average=None, multidim_average=mda,
                                                           ignore_index=ign)
                            else:
                                s = binary_stat_scores(p, tt, threshold=thr, multidim_average=mda, ignore_index=ign)
                            out[f"{key}/ign{ign}/{mda}"] = counts_of(s)
                    case += 1
    out["n_sets"] = np.array(case)
    return out


if __name__ == "__main__":
    data = binary_counts_golden()
    path = os.path.join(HERE, "binary_counts.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB,", len(data), "arrays")
