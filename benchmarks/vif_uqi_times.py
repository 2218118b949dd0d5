"""Kernel K21 (VIF-P and UQI on K20's moments): kernel time, update time and the reference's op chain (oracle/vif.py
`torch_chain_vif`, oracle/uqi.py `torch_chain_uqi`, default torch settings) on the same GPU, with floor bytes and FP32
FLOPs counted from shapes and the bound they give.

  V1  VIF f32  [32, 3, 512, 512], values in 0-255
  V2  VIF bf16 [32, 3, 512, 512], values in 0-255
  V3  VIF f32  [8, 1, 1024, 1024]
  V4  VIF f32  [32, 3, 512, 512] channels-last view
  U1  UQI f32  [32, 3, 512, 512]
  U2  UQI bf16 [32, 3, 512, 512]
  U3  UQI f32  [8, 1, 1024, 1024]
  U4  UQI f32  [32, 3, 512, 512] channels-last view

kernel_us: CUDA events around the `_native` calls of one update (VIF: three decimations and four moment passes; UQI: one
moment pass).  update_us: CUDA events around the functional.  floor_bytes: each pass reads both of its inputs once, a
decimation writes both outputs.  flops: per output position, the five products, 2 · 5 · (taps_h + taps_w) for the
separable filter and 30 for the epilogue; a decimation 2 · 2 · taps² per output (the direct form K21 runs).  bound:
which of bytes / 3.35 TB/s and flops / 67 TFLOP/s (H100 SXM data sheet, 700 W) is larger; share: that time over
kernel_us.  Prints one JSON line with the card name and power limit, read in the same run.
Usage: python benchmarks/vif_uqi_times.py [--iters 10]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from benchmarks.segmentation_times import card, timed  # noqa: E402
from metrics_b200 import _native  # noqa: E402
from metrics_b200.functional.image import uqi as fuqi  # noqa: E402
from metrics_b200.functional.image import vif as fvif  # noqa: E402
from oracle import uqi as ouq  # noqa: E402
from oracle import vif as ovf  # noqa: E402

PEAK_BYTES, PEAK_FLOPS = 3.35e12, 67e12


def inputs(shape, dtype, level, channels_last, seed=0):
    g = torch.Generator().manual_seed(seed)
    p = level * torch.rand(shape, generator=g)
    t = (p + 0.05 * level * torch.randn(shape, generator=g)).clamp(0, level)
    p, t = p.to(dtype).cuda(), t.to(dtype).cuda()
    if channels_last:
        p, t = p.contiguous(memory_format=torch.channels_last), t.contiguous(memory_format=torch.channels_last)
    return p, t


def vif_counts(shape, esize):
    b, c, h, w = shape
    nbytes = flops = 0
    for s, (n, _) in enumerate(fvif.SCALES):
        if s > 0:
            oh, ow = (h - n + 2) // 2, (w - n + 2) // 2
            nbytes += 2 * b * c * (h * w + oh * ow) * esize
            flops += b * c * oh * ow * 2 * 2 * n * n
            h, w = oh, ow
        nbytes += 2 * b * c * h * w * esize
        flops += b * c * (h - n + 1) * (w - n + 1) * (3 + 2 * 5 * 2 * n + 30)
    return nbytes, flops


def workload(name, kind, shape, dtype, channels_last, iters):
    level = 255.0 if kind == "vif" else 1.0
    p, t = inputs(shape, dtype, level, channels_last)
    esize = p.element_size()
    if kind == "vif":
        ws = fvif._scale_weights(dtype, p.device)
        eps, sn = fvif._constants(dtype, 2.0)

        def native():
            x, y = p, t
            for s, (n, _) in enumerate(fvif.SCALES):
                if s > 0:
                    x, y = _native.vif_decimate(x, y, ws[s][1:], (n, n))
                _native.vif_scale(x, y, ws[s], (1, n, n), eps, sn)

        def update():
            return fvif.visual_information_fidelity(p, t)

        def chain():
            return ovf.torch_chain_vif(p, t).mean()
        nbytes, flops = vif_counts(shape, esize)
    else:
        axes = [("u", 1, None), ("g", 11, 1.5), ("g", 11, 1.5)]
        weights = fuqi._weights(axes, dtype, p.device)
        eps = torch.finfo(dtype).eps

        def native():
            _native.uqi(p, t, weights, (1, 11, 11), (0, 5, 5), (5, 5), eps, False)

        def update():
            return fuqi.universal_image_quality_index(p, t)

        def chain():
            return ouq.torch_chain_uqi(p, t).mean()
        b, c, h, w = shape
        nbytes, flops = 2 * b * c * h * w * esize, b * c * h * w * (3 + 2 * 5 * 22 + 30)
    k_s = timed(native, iters)
    u_s = timed(update, iters)
    c_s = timed(chain, max(2, iters // 4))
    t_bytes, t_flops = nbytes / PEAK_BYTES, flops / PEAK_FLOPS
    got, ref = float(update()), float(chain())
    return name, {
        "kernel_us": round(k_s * 1e6, 1), "update_us": round(u_s * 1e6, 1), "chain_us": round(c_s * 1e6, 1),
        "floor_bytes": nbytes, "flops": flops, "bound": "flops" if t_flops > t_bytes else "bytes",
        "share": round(max(t_bytes, t_flops) / k_s, 3), "speedup_vs_chain": round(c_s / k_s, 1),
        "value": got, "chain_value": ref,
    }


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    c = card()
    out = {"card": c["name"], "power_limit_w": c["power_limit_w"], "iters": args.iters}
    with torch.no_grad():
        for spec in (("V1", "vif", (32, 3, 512, 512), torch.float32, False),
                     ("V2", "vif", (32, 3, 512, 512), torch.bfloat16, False),
                     ("V3", "vif", (8, 1, 1024, 1024), torch.float32, False),
                     ("V4", "vif", (32, 3, 512, 512), torch.float32, True),
                     ("U1", "uqi", (32, 3, 512, 512), torch.float32, False),
                     ("U2", "uqi", (32, 3, 512, 512), torch.bfloat16, False),
                     ("U3", "uqi", (8, 1, 1024, 1024), torch.float32, False),
                     ("U4", "uqi", (32, 3, 512, 512), torch.float32, True)):
            name, res = workload(*spec, args.iters)
            out[name] = res
            print(name, json.dumps(res), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
