"""Generate tests/golden/normalize.npz from the UNMODIFIED reference (TorchMetrics under /root/reference), CPU tensors.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_normalize.py

Same import set-up as make_golden.py.  The cases pin `normalize_logits_if_needed` (utilities/compute.py:190-229) for every
float dtype: 1-D sigmoid batches and `[N, C]`, `[N, C, d]` and `[N, C, h, w]` softmax batches, each as logits and as
probabilities; probability batches holding exactly 0, -0.0 and 1; and batches of probabilities with a single score one step
outside [0, 1] (the dtype's smallest negative subnormal, or 1 plus one ulp).  The inputs hold no NaN: the reference's CPU
branch (`all(0 <= x <= 1)`) and device branch (`any(x < 0 | x > 1)`) vote differently only there.
tests/test_oracle_normalize.py replays them through oracle/normalize.py.

The archive is written with fixed zip timestamps, so a rerun reproduces it byte for byte.
"""
from __future__ import annotations

import io
import math
import os
import sys
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "_standins"))
sys.path.insert(0, "/root/reference/src")

from torchmetrics.utilities.compute import normalize_logits_if_needed  # noqa: E402

DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2, torch.float64: 3}
# (smallest positive subnormal, one ulp above 1) of each dtype
STEPS = {torch.float32: (2.0**-149, 2.0**-23), torch.float16: (2.0**-24, 2.0**-10), torch.bfloat16: (2.0**-133, 2.0**-7),
         torch.float64: (2.0**-1074, 2.0**-52)}
SHAPES = {"sigmoid": [(1,), (7,), (100,)], "softmax": [(1, 1), (5, 3), (12, 33), (6, 4, 5), (3, 5, 2, 4)]}


def np_of(t: torch.Tensor) -> np.ndarray:
    """float16 / bfloat16 are stored widened to float32 (exact); the dtype code says what to narrow them back to."""
    return t.float().numpy() if t.dtype in (torch.float16, torch.bfloat16) else t.numpy()


def batches(norm: str, shape, dtype, g: torch.Generator):
    """(kind, input) pairs of one shape and dtype."""
    n = math.prod(shape)
    logits = (torch.randn(n, generator=g, dtype=torch.float64) * 4).to(dtype).reshape(shape)
    if norm == "softmax":
        probs = torch.softmax(torch.randn(shape, generator=g, dtype=torch.float64), 1).to(dtype)
    else:
        probs = torch.rand(n, generator=g, dtype=torch.float64).to(dtype).reshape(shape)
    yield "logits", logits
    yield "probs", probs
    edges = probs.flatten().clone()
    k = min(n, 3)
    edges[torch.randperm(n, generator=g)[:k]] = torch.tensor([0.0, -0.0, 1.0], dtype=dtype)[:k]
    yield "edges", edges.reshape(shape)
    tiny, up = STEPS[dtype]
    for name, v in (("below", -tiny), ("above", 1.0 + up)):
        one = probs.flatten().clone()
        one[int(torch.randint(0, n, (1,), generator=g))] = torch.tensor(v, dtype=torch.float64).to(dtype)
        yield name, one.reshape(shape)


def normalize_golden() -> dict:
    g = torch.Generator().manual_seed(2025)
    out = {}
    case = 0
    for dtype, code in DTYPE_CODE.items():
        for norm, shapes in SHAPES.items():
            for shape in shapes:
                for kind, x in batches(norm, shape, dtype, g):
                    key = f"set{case}"
                    y = normalize_logits_if_needed(x, norm)
                    assert y.dtype == dtype and y.shape == x.shape
                    out[f"{key}/x"] = np_of(x)
                    out[f"{key}/y"] = np_of(y)
                    out[f"{key}/meta"] = np.array([code, int(norm == "softmax")])
                    out[f"{key}/kind"] = np.array(kind)
                    case += 1
    out["n_sets"] = np.array(case)
    return out


def write_npz(path: str, data: dict) -> None:
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(data):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(data[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


if __name__ == "__main__":
    data = normalize_golden()
    path = os.path.join(HERE, "normalize.npz")
    write_npz(path, data)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB,", len(data), "arrays")
