"""Kernel K20 (structural similarity): kernel time, update time, floor bytes and FP32 FLOPs counted from shapes, the
share of the larger of the two bounds, the reference's op chain (oracle/ssim.py `torch_chain_ssim`, default torch
settings) on the same GPU, and the largest deviation of the chain and of K20 from the float64 oracle.

  W1  f32 [16, 3, 512, 512], data_range=1.0
  W2  W1 with data_range=None (adds the data-range pre-pass; the chain synchronises the host there)
  W3  bf16 [8, 3, 1024, 1024], data_range=1.0
  W4  MS-SSIM f32 [8, 3, 512, 512], data_range=1.0 (five scales; the chain runs its own pool between them)
  W5  3-D f32 [2, 1, 64, 128, 128], data_range=1.0

kernel_us: CUDA events around the `_native` calls of one update (pre-pass, K20, pools).  update_us: CUDA events around
the functional.  floor_bytes: both inputs read once per scale.  flops: per output position and channel, the five
products and 2 · 5 · (taps_d + taps_h + taps_w) for the separable filter, plus 20 for the epilogue.  bound: which of
bytes / 3.35 TB/s and flops / 67 TFLOP/s (H100 SXM data sheet, 700 W) is larger; share: that time over kernel_us.
max_dev_*: largest per-image deviation from the oracle (taps of weight 1, as K20 uses them), over the first two images.
Prints one JSON line with the card name and power limit, read in the same run.
Usage: python benchmarks/ssim_times.py [--iters 20]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from benchmarks.segmentation_times import card, timed  # noqa: E402
from metrics_b200 import _native  # noqa: E402
from metrics_b200.functional.image import ssim as fssim  # noqa: E402
from oracle import ssim as osm  # noqa: E402

PEAK_BYTES, PEAK_FLOPS = 3.35e12, 67e12
BETAS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)


def inputs(shape, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    p = torch.rand(shape, generator=g)
    t = (p + 0.05 * torch.randn(shape, generator=g)).clamp(0, 1)
    return p.to(dtype).cuda(), t.to(dtype).cuda()


def scales(shape, n):
    out = [list(shape)]
    for _ in range(n - 1):
        out.append(out[-1][:2] + [s // 2 for s in out[-1][2:]])
    return out


def counts(shape, dtype, taps):
    px = int(np.prod(shape))
    flops = px * (3 + 2 * 5 * sum(taps) + 20)
    return 2 * px * torch.tensor([], dtype=dtype).element_size(), flops


def chain_ms(p, t, data_range):
    vals = []
    for k in range(len(BETAS)):
        s, cs, _ = osm.torch_chain_ssim(p, t, data_range=data_range)
        vals.append(torch.relu(s if k == len(BETAS) - 1 else cs))
        p, t = torch.nn.functional.avg_pool2d(p, 2), torch.nn.functional.avg_pool2d(t, 2)
    b = torch.tensor(BETAS, device=p.device).view(-1, 1)
    return torch.prod(torch.stack(vals) ** b, 0)


def workload(name, shape, dtype, data_range, ms, kw, iters):
    p, t = inputs(shape, dtype, 0)
    axes, _ = osm.plan(len(shape), True, kw.get("sigma", 1.5), kw.get("kernel_size", 11))
    taps = [a[1] for a in axes] if len(shape) == 5 else [1] + [a[1] for a in axes]
    if ms:
        def native():
            x, y = p, t
            for k in range(len(BETAS)):
                fssim._ssim_scale(x, y, True, [1.5, 1.5], [11, 11], data_range, 0.01, 0.03, True, False)
                if k < len(BETAS) - 1:
                    x, y = _native.ssim_avg_pool(x, y, False)

        def update():
            return fssim.multiscale_structural_similarity_index_measure(p, t, data_range=data_range, reduction="none")

        def chain():
            return chain_ms(p, t, data_range)
        shapes = scales(shape, len(BETAS))
    else:
        ks, sg = kw.get("kernel_size", 11), kw.get("sigma", 1.5)
        n = len(shape) - 2
        ks = list(ks) if isinstance(ks, (list, tuple)) else [ks] * n
        sg = list(sg) if isinstance(sg, (list, tuple)) else [sg] * n

        def native():
            fssim._ssim_scale(p, t, True, sg, ks, data_range, 0.01, 0.03, False, False)

        def update():
            return fssim.structural_similarity_index_measure(p, t, data_range=data_range, reduction="none", **kw)

        def chain():
            return osm.torch_chain_ssim(p, t, data_range=data_range, **kw)[0]
        shapes = [shape]
    nbytes = flops = 0
    for s in shapes:
        b, f = counts(s, dtype, taps)
        nbytes, flops = nbytes + b, flops + f
    k_s = timed(native, iters)
    u_s = timed(update, iters)
    c_s = timed(chain, max(3, iters // 4))
    t_bytes, t_flops = nbytes / PEAK_BYTES, flops / PEAK_FLOPS
    got, ref = update()[:2].double().cpu().numpy(), chain()[:2].double().cpu().numpy()
    pn, tn = p[:2].double().cpu().numpy(), t[:2].double().cpu().numpy()
    wtaps = osm.filter_taps(axes, dtype, "cuda")
    if ms:
        want = osm.ms_ssim(pn, tn, data_range=data_range, taps=wtaps, round_to=dtype, unit_taps=True)
    else:
        want = osm.ssim(pn, tn, data_range=data_range, taps=wtaps, unit_taps=True, **kw)[0]
    return name, {
        "kernel_us": round(k_s * 1e6, 1), "update_us": round(u_s * 1e6, 1), "chain_us": round(c_s * 1e6, 1),
        "floor_bytes": nbytes, "flops": flops, "bound": "flops" if t_flops > t_bytes else "bytes",
        "share": round(max(t_bytes, t_flops) / k_s, 3), "speedup_vs_chain": round(c_s / k_s, 1),
        "max_dev_k20": float(np.abs(got - want).max()), "max_dev_chain": float(np.abs(ref - want).max()),
    }


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    c = card()
    out = {"card": c["name"], "power_limit_w": c["power_limit_w"], "iters": args.iters}
    with torch.no_grad():
        for spec in (("W1", (16, 3, 512, 512), torch.float32, 1.0, False, {}),
                     ("W2", (16, 3, 512, 512), torch.float32, None, False, {}),
                     ("W3", (8, 3, 1024, 1024), torch.bfloat16, 1.0, False, {}),
                     ("W4", (8, 3, 512, 512), torch.float32, 1.0, True, {}),
                     ("W5", (2, 1, 64, 128, 128), torch.float32, 1.0, False, {})):
            name, res = workload(*spec, args.iters)
            out[name] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
