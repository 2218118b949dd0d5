"""Inputs of the Hausdorff-distance goldens (tests/golden/hausdorff.npz, made by tests/golden/make_golden_hausdorff.py)
and the helpers the CPU and GPU tests share: the case table, the class / functional replay, and a stand-in of
`_native.hausdorff_distance` built on the numpy oracle."""
from __future__ import annotations

import os

import numpy as np
import torch

from oracle import hausdorff as oh

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "hausdorff.npz")
METRICS = ("euclidean", "chessboard", "taxicab")
SPACINGS = (None, [2, 3], [0.7, 1.3], [1, 0.37])
ONE_HOT_DTYPES = (torch.bool, torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64)


def blobs(rng: np.random.Generator, n: int, c: int, side: int, density: float = 0.25) -> np.ndarray:
    """``[n, c, side, side]`` bool masks: a few rectangles plus sparse noise, never empty."""
    out = rng.random((n, c, side, side)) < density / 8
    for b in range(n):
        for k in range(c):
            for _ in range(int(rng.integers(1, 4))):
                r0, c0 = rng.integers(0, side, 2)
                out[b, k, r0:r0 + int(rng.integers(1, side // 2 + 2)), c0:c0 + int(rng.integers(1, side // 2 + 2))] = True
    return out


def cases() -> list[dict]:
    """Every golden case: name, two batches of numpy inputs, keyword arguments of the reference call."""
    rng = np.random.default_rng(2024)
    out = []
    for metric in METRICS:
        for si, spacing in enumerate(SPACINGS):
            for directed in (False, True):
                p, t = blobs(rng, 4, 3, 24), blobs(rng, 4, 3, 24)
                out.append(dict(name=f"onehot_{metric}_s{si}_{'dir' if directed else 'sym'}", preds=p.astype(np.int64),
                                target=t.astype(np.int64), kwargs=dict(num_classes=3, distance_metric=metric,
                                                                        spacing=spacing, directed=directed)))
    for bg in (False, True):
        lab = rng.integers(0, 4, (4, 20, 20))
        lab2 = np.roll(lab, 2, axis=2)
        out.append(dict(name=f"index_bg{int(bg)}", preds=lab, target=lab2,
                        kwargs=dict(num_classes=4, include_background=bg, input_format="index", spacing=[0.7, 1.3])))
    for dt in ONE_HOT_DTYPES:
        p, t = blobs(rng, 4, 3, 20), blobs(rng, 4, 3, 20)
        out.append(dict(name=f"dtype_{str(dt).split('.')[-1]}", preds=p, target=t, dtypes=(dt, dt),
                        kwargs=dict(num_classes=3, include_background=True)))
    p, t = blobs(rng, 4, 3, 20), blobs(rng, 4, 3, 20)
    out.append(dict(name="dtype_mixed", preds=p, target=t, dtypes=(torch.uint8, torch.int32),
                    kwargs=dict(num_classes=3, distance_metric="taxicab")))
    p, t = blobs(rng, 4, 3, 16), blobs(rng, 4, 3, 16)
    p[1, 2] = False
    t[2, 1] = False
    for directed in (False, True):
        out.append(dict(name=f"one_side_empty_{'dir' if directed else 'sym'}", preds=p.astype(np.int64),
                        target=t.astype(np.int64), kwargs=dict(num_classes=3, directed=directed)))
    p, t = blobs(rng, 4, 2, 48, 0.05), blobs(rng, 4, 2, 48, 0.05)
    out.append(dict(name="side48", preds=p.astype(np.int64), target=t.astype(np.int64),
                    kwargs=dict(num_classes=2, include_background=True)))
    return out


def tensors(case: dict, device="cpu"):
    """The case's two batches as tensors: (preds, target) and the same pair with preds and target swapped."""
    dp, dt = case.get("dtypes", (torch.int64, torch.int64))
    p = torch.from_numpy(np.ascontiguousarray(case["preds"])).to(dp).to(device)
    t = torch.from_numpy(np.ascontiguousarray(case["target"])).to(dt).to(device)
    return [(p, t), (t.to(dp), p.to(dt))]


def load() -> dict:
    return dict(np.load(GOLDEN))


def ulps(got: np.ndarray, want: np.ndarray) -> int:
    """Largest distance in float32 units in the last place between two non-negative float32 arrays (inf included)."""
    return int(np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64)).max(initial=0))


def golden_ulps(case: dict) -> int:
    """How far a golden distance may be from the correctly rounded one: the reference's euclidean distances on CPU
    tensors come from torch's vectorised float32 sqrt, which is not always correctly rounded (one unit in the last
    place); K19 and the oracle round sqrt correctly, as torch does on CUDA tensors.  Other metrics are bit-equal."""
    return 1 if case["kwargs"].get("distance_metric", "euclidean") == "euclidean" else 0


def check_case(golden: dict, case: dict, device) -> None:
    """Functional on the first batch and the class over both batches against the goldens: bit for bit but for the
    reference's CPU sqrt (`golden_ulps`)."""
    from metrics_b200.functional.segmentation import hausdorff_distance
    from metrics_b200.segmentation import HausdorffDistance

    name, kw = case["name"], case["kwargs"]
    batches = tensors(case, device)
    got = hausdorff_distance(*batches[0], **kw)
    want = golden[f"{name}/functional"]
    assert got.dtype == torch.float32 and got.device.type == torch.device(device).type
    assert ulps(got.cpu().numpy(), want) <= golden_ulps(case), (name, got, want)
    m = HausdorffDistance(**kw).to(device)
    for p, t in batches:
        m.update(p, t)
    # the distances are exact; `score` is torch's float32 sum of them, whose order differs between CPU and CUDA
    exact = torch.device(device).type == "cpu" and golden_ulps(case) == 0
    for state in ("score", "total", "compute"):
        g = (m.compute() if state == "compute" else getattr(m, state)).cpu().numpy()
        w = golden[f"{name}/{state}"]
        same = np.array_equal(g, w) if exact or state == "total" else np.allclose(g, w, rtol=1e-6, atol=0)
        assert g.dtype == w.dtype and same, (name, state, g, w)


def standin(preds, target, num_classes, index_format, drop_background, distance_metric, spacing, directed):
    """`_native.hausdorff_distance` on CPU tensors from the numpy oracle: same outputs, same error word."""
    p, t = preds.numpy(), target.numpy()
    labels = 0
    if index_format:
        for x, neg, big in ((p, 1, 2), (t, 4, 8)):
            labels |= (neg if (x < 0).any() else 0) | (big if (x >= num_classes).any() else 0)
        c = num_classes
        p = np.stack([p == k for k in range(c)], 1)
        t = np.stack([t == k for k in range(c)], 1)
    c = p.shape[1]
    off = 1 if drop_background and c > 1 else 0
    out = np.zeros((p.shape[0], c - off), np.float32)
    code = -1
    for b in range(p.shape[0]):
        for k in range(c - off):
            q = b * (c - off) + k
            pm, tm = p[b, k + off], t[b, k + off]
            bad = [not np.isin(x, (0, 1)).all() for x in (pm, tm)]
            d = None if any(bad) else oh.pair_distance(pm != 0, tm != 0, spacing, distance_metric, directed)
            if code < 0 and (any(bad) or d is None):
                code = 4 * q + (0 if bad[0] else 1 if bad[1] else 2)
            out[b, k] = 0 if d is None else d
    return torch.from_numpy(out), torch.tensor([code, labels], dtype=torch.int64)
