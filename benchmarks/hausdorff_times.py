"""Kernel K19 (Hausdorff distance): kernel time and `update()` time per call, the distances against the numpy oracle, and
the reference's pytorch-engine op chain (oracle/hausdorff.py `chain_pair`) on the same GPU for comparison.

  W1  int64 labels [32, 512, 512], 4 classes, background dropped: ellipses with perturbed boundaries; preds shifted
  W2  int64 labels [8, 1024, 1024], 19 classes, every class present in every frame (horizontal bands with wavy borders,
      so the reference would not raise); preds shifted
  W3  bool one-hot [16, 3, 512, 512], spacing [0.8, 1.25]: ellipses per channel
  W4  the row scan's worst case at 512 x 512: a checkerboard pred (every pixel of it an edge) against a 16 x 16 corner
      blob target, 4 images

kernel_us: CUDA events around the C-ABI call (memsets and two kernels per scratch launch).  update_us: host clock around
`HausdorffDistance.update()`, which ends in its one host synchronisation.  floor_bytes: both inputs read once.
distances_equal: the kernel's [N, C'] against the oracle, on the first sample (the oracle is numpy on the CPU).
chain_us_per_pair: the op chain on a prefix of pairs whose dense [pixels, edge pixels] temporaries stay under 8 GB,
chain_pairs of them (0 when the first pair alone would exceed it).  Prints one JSON line with the card name and power
limit, read in the same run.  Usage: python benchmarks/hausdorff_times.py [--iters 10]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from benchmarks.segmentation_times import card, timed  # noqa: E402

CHAIN_BYTES = 8e9
CHAIN_MAX_PAIRS = 4


def ellipses(g, n, k, h, w):
    """int64 [n, h, w] labels 0..k-1: k - 1 ellipses per image over background 0, one per horizontal strip so that none
    hides another (every class is present), boundaries perturbed by a sine."""
    i = torch.arange(h).view(h, 1).float()
    j = torch.arange(w).view(1, w).float()
    lab = torch.zeros(n, h, w, dtype=torch.int64)
    strip = h / (k - 1)
    for b in range(n):
        for c in range(1, k):
            u = torch.rand(4, generator=g)
            cy, cx = (c - 0.5 + 0.2 * (u[0] - 0.5)) * strip, w * (0.3 + 0.4 * u[1])
            ry, rx = strip * (0.15 + 0.2 * u[2]), w * (0.1 + 0.15 * u[3])
            ang = torch.atan2(i - cy, j - cx)
            r = 1 + 0.08 * torch.sin(7 * ang + float(torch.rand(1, generator=g)) * 6)
            lab[b][((i - cy) / ry) ** 2 + ((j - cx) / rx) ** 2 < r ** 2] = c
    return lab


def bands(g, n, k, h, w):
    """int64 [n, h, w]: k horizontal bands with wavy borders, every class present in every frame."""
    j = torch.arange(w).float()
    lab = torch.empty(n, h, w, dtype=torch.int64)
    i = torch.arange(h).view(h, 1).float()
    for b in range(n):
        phase = float(torch.rand(1, generator=g)) * 6
        edges = [(c + 1) * h / k + 6 * torch.sin(j / 17 + phase + c) for c in range(k - 1)]
        lab[b] = sum((i >= e.view(1, w)).long() for e in edges)
    return lab


def workloads():
    g = torch.Generator().manual_seed(2026)
    t1 = ellipses(g, 32, 4, 512, 512)
    t2 = bands(g, 8, 19, 1024, 1024)
    t3 = torch.stack([ellipses(g, 16, 2, 512, 512) == 1 for _ in range(3)], 1)
    i, j = torch.meshgrid(torch.arange(512), torch.arange(512), indexing="ij")
    board = ((i + j) % 2 == 0).expand(4, 1, 512, 512).contiguous()
    blob = torch.zeros_like(board)
    blob[..., :16, :16] = True
    return {
        "W1": (torch.roll(t1, (3, -5), (1, 2)), t1, dict(num_classes=4, input_format="index")),
        "W2": (torch.roll(t2, (4, 7), (1, 2)), t2, dict(num_classes=19, include_background=True, input_format="index")),
        "W3": (torch.roll(t3, (2, 3), (2, 3)), t3, dict(num_classes=3, include_background=True, spacing=[0.8, 1.25])),
        "W4": (board, blob, dict(num_classes=1, include_background=True)),
    }


def one_hot_pairs(p, t, kw):
    """Per pair (b, c) the two bool masks, in the kernel's pair order."""
    if kw.get("input_format") == "index":
        p = torch.nn.functional.one_hot(p, kw["num_classes"]).movedim(-1, 1)
        t = torch.nn.functional.one_hot(t, kw["num_classes"]).movedim(-1, 1)
    if not kw.get("include_background", False) and p.shape[1] > 1:
        p, t = p[:, 1:], t[:, 1:]
    return p.bool(), t.bool()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from metrics_b200 import _native
    from metrics_b200.segmentation import HausdorffDistance
    from oracle import hausdorff as oh

    dev = torch.device("cuda:0")
    result = {"card": None, "power_limit_w": None, "iters": args.iters}
    info = card()
    result["card"], result["power_limit_w"] = info["name"], info["power_limit_w"]
    for name, (p_cpu, t_cpu, kw) in workloads().items():
        p, t = p_cpu.to(dev), t_cpu.to(dev)
        index = kw.get("input_format") == "index"
        spacing = kw.get("spacing") or [1, 1]
        sp = [v if isinstance(v, int) else float(v) for v in spacing]

        def call():
            return _native.hausdorff_distance(p, t, kw["num_classes"], index, not kw.get("include_background", False),
                                              "euclidean", sp, False)

        kernel_s = timed(call, args.iters)
        m = HausdorffDistance(**kw).to(dev)
        m.update(p, t)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.iters):
            m.update(p, t)
        update_s = (time.perf_counter() - t0) / args.iters
        out, err = call()
        assert err.tolist() == [-1, 0], err
        want = oh.hausdorff(p_cpu[:1].numpy(), t_cpu[:1].numpy(), kw["num_classes"], kw.get("include_background", False),
                            "euclidean", kw.get("spacing"), False, kw.get("input_format", "one-hot"))
        equal = bool(torch.equal(out[:1].cpu(), torch.from_numpy(want)))
        pm, tm = one_hot_pairs(p_cpu, t_cpu, kw)
        pm, tm = pm.flatten(0, 1), tm.flatten(0, 1)
        h, w = pm.shape[-2:]
        pairs = 0
        for q in range(min(CHAIN_MAX_PAIRS, pm.shape[0])):
            edges = max(int(oh.edges(pm[q].numpy()).sum()), int(oh.edges(tm[q].numpy()).sum()))
            if (h + 2) * (w + 2) * edges * 40 > CHAIN_BYTES:  # int64 dr, dc, their products and the float32 results
                break
            pairs += 1
        chain_us = None
        if pairs:
            pg, tg = pm[:pairs].to(dev), tm[:pairs].to(dev)
            oh.chain_pair(pg[0], tg[0], spacing, "euclidean", False)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            t0 = time.perf_counter()
            for q in range(pairs):
                oh.chain_pair(pg[q], tg[q], spacing, "euclidean", False)
            torch.cuda.synchronize()
            chain_us = round((time.perf_counter() - t0) / pairs * 1e6, 1)
        floor = p.numel() * p.element_size() + t.numel() * t.element_size()
        result[name] = {"kernel_us": round(kernel_s * 1e6, 1), "update_us": round(update_s * 1e6, 1), "floor_bytes": floor,
                        "pairs": out.numel(), "distances_equal": equal, "chain_us_per_pair": chain_us,
                        "chain_pairs": pairs}
        del p, t
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
