"""Kernel K15 (segmentation overlap counts): kernel time and `update()` time per call in a stream of updates, against the
reference's op chain (oracle/segmentation.py: one_hot + movedim, `&` / `*`, three sums) on the same GPU and tensors.

  W1  MeanIoU(19, input_format="index"), int64 [8, 1024, 2048]; targets a random [8, 32, 64] map upsampled x32 (nearest),
      preds the targets with about 10% of the 32 x 32 blocks relabelled
  W2  W1's shape with uniform random labels: no same-class runs, so a warp of 32 pixels holds about 15 of the 19 classes
      and the warp aggregation takes its __match_any_sync path instead of the all-lanes-equal one
  W3  DiceScore(21), bool one-hot [16, 21, 512, 512], planar and channels-last; the same in float16 at N = 16 and N = 1
      (float sums are split over many CTAs and folded in a fixed order)
  W4  GeneralizedDiceScore(150, input_format="index"), int64 [16, 512, 512]

Prints one JSON line with the card name and power limit, read in the same run.  Usage:
python benchmarks/segmentation_times.py [--iters 20]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

PEAK_BW = {"NVIDIA H100 80GB HBM3": 3.35e12}  # data-sheet HBM bandwidth by driver name (H100 SXM)


def card() -> dict:
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        power = None
    return {"name": name, "power_limit_w": power}


def timed(fn, iters: int, warmup: int = 3) -> float:
    """Mean seconds per call over `iters` back-to-back calls between two CUDA events (after `warmup` untimed calls)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / 1e3 / iters


def workloads(dev):
    g = torch.Generator(device=dev).manual_seed(2026)
    small = torch.randint(0, 19, (8, 32, 64), generator=g, device=dev)
    t1 = small.repeat_interleave(32, 1).repeat_interleave(32, 2).contiguous()
    relabel = (torch.rand((8, 32, 64), generator=g, device=dev) < 0.1)
    p_small = torch.where(relabel, torch.randint(0, 19, (8, 32, 64), generator=g, device=dev), small)
    p1 = p_small.repeat_interleave(32, 1).repeat_interleave(32, 2).contiguous()
    p2 = torch.randint(0, 19, (8, 1024, 2048), generator=g, device=dev)
    t2 = torch.randint(0, 19, (8, 1024, 2048), generator=g, device=dev)
    lab3p = torch.randint(0, 21, (16, 512, 512), generator=g, device=dev)
    lab3t = torch.randint(0, 21, (16, 512, 512), generator=g, device=dev)
    cl3 = [torch.nn.functional.one_hot(x, 21).bool().movedim(-1, 1) for x in (lab3p, lab3t)]
    pl3 = [x.contiguous() for x in cl3]
    cl3h = [x.half() for x in cl3]  # .half() keeps the channels-last strides
    pl3h = [x.contiguous() for x in cl3h]
    del lab3p, lab3t
    p4 = torch.randint(0, 150, (16, 512, 512), generator=g, device=dev)
    t4 = torch.randint(0, 150, (16, 512, 512), generator=g, device=dev)
    return [
        ("W1", "MeanIoU", dict(num_classes=19, input_format="index"), p1, t1, 2 * 8 * 2**21 * 8),
        ("W2", "MeanIoU", dict(num_classes=19, input_format="index"), p2, t2, 2 * 8 * 2**21 * 8),
        ("W3_planar", "DiceScore", dict(num_classes=21), pl3[0], pl3[1], 2 * 16 * 21 * 2**18),
        ("W3_channels_last", "DiceScore", dict(num_classes=21), cl3[0], cl3[1], 2 * 16 * 21 * 2**18),
        ("W3_f16_planar", "DiceScore", dict(num_classes=21), pl3h[0], pl3h[1], 2 * 16 * 21 * 2**18 * 2),
        ("W3_f16_channels_last", "DiceScore", dict(num_classes=21), cl3h[0], cl3h[1], 2 * 16 * 21 * 2**18 * 2),
        ("W3_f16_planar_n1", "DiceScore", dict(num_classes=21), pl3h[0][:1], pl3h[1][:1], 2 * 21 * 2**18 * 2),
        ("W3_f16_channels_last_n1", "DiceScore", dict(num_classes=21), cl3h[0][:1], cl3h[1][:1], 2 * 21 * 2**18 * 2),
        ("W4", "GeneralizedDiceScore", dict(num_classes=150, input_format="index"), p4, t4, 2 * 16 * 2**18 * 8),
    ]


def chain_states(kind, kw, p, t):
    from oracle import segmentation as osg

    index = kw.get("input_format") == "index"
    c = kw["num_classes"]
    if kind == "MeanIoU":
        return osg.mean_iou_chain(p, t, c, True, False, index).mean().reshape(1), None
    if kind == "DiceScore":
        return None, osg.dice_update_chain(p, t, c, True, index)
    return osg.generalized_dice_chain(p, t, c, True, "square", False, index).sum(0).reshape(1), None


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from metrics_b200 import _native, segmentation

    dev = torch.device("cuda:0")
    info = card()
    peak = PEAK_BW.get(info["name"])
    rows = {}
    for name, kind, kw, p, t, floor in workloads(dev):
        index = kw.get("input_format") == "index"
        mul = kind != "MeanIoU"
        flag = torch.zeros(1, dtype=torch.int32, device=dev) if index else None
        kernel_s = timed(lambda: _native.segmentation_overlap_counts(p, t, kw["num_classes"], index, mul, False, flag), args.iters)
        metric = getattr(segmentation, kind)(**kw).to(dev)

        def update():
            metric.update(p, t)
            if kind == "DiceScore" and len(metric.numerator) > 8:  # keep the cat states small in a long stream
                metric.reset()

        update_s = timed(update, args.iters)
        from oracle import segmentation as osg

        c = kw["num_classes"]
        chain_s = timed(lambda: osg.counts_chain(p, t, c, True, index, "mul" if mul else "and"), max(3, args.iters // 4), 1)
        # equality: counts bit for bit, the per-batch float state within 1e-6
        counts = _native.segmentation_overlap_counts(p, t, c, index, mul, False, flag)
        want = osg.counts_chain(p, t, c, True, index, "mul" if mul else "and")
        # float counts are float64 sums rounded once to the input dtype by the metrics; compare them that way
        counts_equal = all(torch.equal(counts[k].to(want[k].dtype), want[k]) for k in range(3))
        fresh = getattr(segmentation, kind)(**kw).to(dev)
        fresh.update(p, t)
        score, dice = chain_states(kind, kw, p, t)
        if dice is not None:
            states_equal = all(torch.equal(getattr(fresh, s)[0], w) for s, w in zip(("numerator", "denominator", "support"), dice))
        else:
            states_equal = bool(torch.allclose(fresh.score, score, rtol=1e-6, atol=0))
        row = {"kernel_us": round(kernel_s * 1e6, 1), "update_us": round(update_s * 1e6, 1),
               "chain_us": round(chain_s * 1e6, 1), "floor_bytes": floor,
               "kernel_tb_s": round(floor / kernel_s / 1e12, 3), "counts_equal": counts_equal, "states_equal": states_equal}
        if not index:
            row["layout"] = ("planar", "channels_last")[_native._one_hot_layout(p)[0]]
        if peak:
            row["share_of_peak"] = round(floor / kernel_s / peak, 3)
        rows[name] = row
        del metric, fresh
        torch.cuda.empty_cache()
    print(json.dumps({"card": info["name"], "power_limit_w": info["power_limit_w"], "iters": args.iters, **rows}))


if __name__ == "__main__":
    main()
