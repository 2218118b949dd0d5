"""Kernel K18 (panoptic quality): kernel time and `update()` time per call, against the torch op chain of
oracle/panoptic.py (three torch.unique(dim=0) per image, then the matching rules as tensor ops) on the same GPU and tensors.
The chain leaves out the reference's per-pair Python loop, so it is a lower bound on the reference's time.

  W1  Cityscapes-like: PanopticQuality, int64 [8, 1024, 2048, 2], 8 things and 11 stuffs, 128 regions of 128 x 128 per
      frame (about 100 segments: stuff regions of one category merge); preds are the targets with every region boundary
      shifted, the instance ids relabelled and about 3% of the regions an unknown category
  W2  COCO-like: PanopticQuality, int32 [32, 640, 640, 2], 80 things and 53 stuffs, 100 regions of 64 x 64 per frame
  W3  pathological: ModifiedPanopticQuality, int64 [2, 512, 512, 2], a distinct instance on every pixel: the first pass's
      tables overflow and every update is counted again with tables of 2 * pixels slots

kernel_us: CUDA events around the C-ABI call alone (memsets and five kernels; the first pass for W3, then the repeat).
update_us: host clock around `update()`, which ends in its one host synchronisation.  Prints one JSON line with the card
name and power limit, read in the same run.  Usage: python benchmarks/panoptic_times.py [--iters 20]
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

from benchmarks.segmentation_times import PEAK_BW, card, timed  # noqa: E402

CITY_THINGS, CITY_STUFFS = list(range(24, 32)), [7, 8, 11, 12, 13, 17, 19, 20, 21, 22, 23]
COCO_THINGS, COCO_STUFFS = list(range(1, 81)), list(range(92, 145))


def regions(g, dev, b, h, w, block, things, stuffs, unknown_frac=0.0):
    """[b, h, w, 2] int64: a grid of block x block regions, each a random category; thing regions get distinct instances."""
    gh, gw = h // block, w // block
    cats = torch.tensor(things + stuffs, device=dev)
    cat = cats[torch.randint(0, len(cats), (b, gh, gw), generator=g, device=dev)]
    if unknown_frac:
        cat = torch.where(torch.rand(cat.shape, generator=g, device=dev) < unknown_frac, torch.full_like(cat, 255), cat)
    inst = torch.arange(gh * gw, device=dev).view(1, gh, gw).expand(b, gh, gw) + 1
    x = torch.stack([cat, inst], -1).repeat_interleave(block, 1).repeat_interleave(block, 2)
    return x.contiguous()


def shifted(g, dev, t, dy, dx):
    """Boundaries moved by (dy, dx), instances relabelled by a fixed permutation."""
    p = torch.roll(t, (dy, dx), (1, 2)).clone()
    perm = torch.randperm(int(t[..., 1].max()) + 1, generator=g, device=dev)
    p[..., 1] = perm[p[..., 1]]
    return p


def workloads(dev):
    g = torch.Generator(device=dev).manual_seed(2026)
    t1 = regions(g, dev, 8, 1024, 2048, 128, CITY_THINGS, CITY_STUFFS)
    p1 = regions(g, dev, 8, 1024, 2048, 128, CITY_THINGS, CITY_STUFFS, unknown_frac=0.03)
    p1 = shifted(g, dev, torch.where((p1[..., :1] == 255), p1, t1), 5, 9)
    t2 = regions(g, dev, 32, 640, 640, 64, COCO_THINGS, COCO_STUFFS).int()
    p2 = shifted(g, dev, t2.long(), 3, 4).int()
    t3 = torch.stack([torch.ones(2, 512, 512, dtype=torch.int64, device=dev),
                      torch.randperm(2 * 512 * 512, generator=g, device=dev).view(2, 512, 512)], -1)
    p3 = torch.roll(t3, 1, 2).contiguous()
    return {
        "W1": (p1, t1, CITY_THINGS, CITY_STUFFS, False, True),
        "W2": (p2, t2, COCO_THINGS, COCO_STUFFS, False, False),
        "W3": (p3, t3, [1], [2], True, False),
    }


def device_calls(_native, states, p, t, cats, n_things, modified, allow):
    """The C-ABI calls of one update without its host synchronisation: the first pass and, when it overflows (W3), the
    repeat with tables of 2 * pixels slots, each with its scratch allocated up front."""
    lib, dev = _native.lib(), p.device
    n, pixels, k = p.shape[0], p[0].numel() // 2, cats.numel() // 2
    worst = _native._pow2_at_least(2 * pixels)
    err = torch.zeros(1, dtype=torch.int32, device=dev)

    def alloc(per, cc, pcap):
        return torch.empty(lib.mb200_panoptic_scratch_bytes(n, pixels, k, per, cc, pcap, _native.tag(p), _native.tag(t)),
                           dtype=torch.uint8, device=dev)

    def run(passes, bufs):
        for (per, cc, pcap), scratch in zip(passes, bufs):
            rc = lib.mb200_panoptic_update(p.data_ptr(), _native.tag(p), t.data_ptr(), _native.tag(t), n, pixels, cats.data_ptr(),
                                           k, n_things, int(modified), int(allow), per, cc, pcap, *[s.data_ptr() for s in states],
                                           scratch.data_ptr(), scratch.numel(), err.data_ptr(), _native.stream_handle(dev))
            _native.check(rc, "panoptic_update")

    passes = [(n, min(_native.PANOPTIC_COLOR_CAPACITY, worst), min(_native.PANOPTIC_PAIR_CAPACITY, worst))]
    run(passes, [alloc(*passes[0])])
    if int(err.item()) & _native.FLAG_CAPACITY:
        per_image = int(lib.mb200_panoptic_scratch_bytes(1, pixels, k, 1, worst, worst, _native.tag(p), _native.tag(t)))
        passes.append((max(1, min(n, _native.PANOPTIC_RERUN_BYTES // per_image)), worst, worst))
    bufs = [alloc(*ps) for ps in passes]
    return lambda: run(passes, bufs)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from metrics_b200 import _native
    from metrics_b200.detection import ModifiedPanopticQuality, PanopticQuality
    from oracle import panoptic as op

    dev = torch.device("cuda:0")
    info = card()
    out = {"card": info["name"], "power_limit_w": info["power_limit_w"], "iters": args.iters}
    peak = PEAK_BW.get(info["name"])
    for name, (p, t, things, stuffs, modified, allow) in workloads(dev).items():
        cls = ModifiedPanopticQuality if modified else PanopticQuality
        m = cls(things, stuffs, allow_unknown_preds_category=allow).to(dev)
        m.update(p, t)
        chain = op.chain_update(p, t, set(things), set(stuffs), modified)
        torch.cuda.synchronize()
        equal = all(torch.equal(a, b) for a, b in zip((m.iou_sum, m.true_positives, m.false_positives, m.false_negatives), chain))
        cats = _native.panoptic_categories(set(things), set(stuffs), dev)
        states = [s.clone() for s in (m.iou_sum, m.true_positives, m.false_positives, m.false_negatives)]
        kernel_s = timed(device_calls(_native, states, p, t, cats, len(things), modified, allow), args.iters)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.iters):
            m.update(p, t)
        torch.cuda.synchronize()
        update_s = (time.perf_counter() - t0) / args.iters
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        op.chain_update(p, t, set(things), set(stuffs), modified)
        torch.cuda.synchronize()
        chain_s = time.perf_counter() - t0
        floor = p.numel() * p.element_size() + t.numel() * t.element_size()
        row = {"kernel_us": round(kernel_s * 1e6, 1), "update_us": round(update_s * 1e6, 1), "chain_us": round(chain_s * 1e6, 1),
               "floor_bytes": floor, "kernel_tb_s": round(floor / kernel_s / 1e12, 3), "states_equal": equal}
        if peak:
            row["share_of_peak"] = round(floor / peak / kernel_s, 3)
        out[name] = row
    print(json.dumps(out))


if __name__ == "__main__":
    main()
