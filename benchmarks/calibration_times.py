"""Calibration error (K14) on one GPU: prints ONE JSON line.

  update   MulticlassCalibrationError(num_classes=1000).update on the seed-0 [65536, 1000] bf16 logits of bench.py's cfg2
           (same recipe: CPU generator seed 0, randn -> bf16, uniform int64 labels), CUDA-event time per call, against the
           algorithmic HBM floor (one read of the logits and the targets, one write of the two float32 states: N*C*2 + N*8
           + N*8 = 132 120 576 B) and the data-sheet bandwidth of the card when it is known (H100 SXM: 3.35 TB/s).
  chain    the reference's op chain (normalize_logits_if_needed -> max -> eq -> float, oracle/calibration.py) on the same GPU
           and tensors; its states are compared with K14a's bit for bit.
  compute  compute() at N = 10**7 confidences, n_bins=15 (K14b + epilogue), against the reference's compute chain.

The card name and power limit are read in the same run.  Usage: python benchmarks/calibration_times.py [--iters 50]
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

N_ROWS, N_CLASSES = 65536, 1000
FLOOR_BYTES = N_ROWS * N_CLASSES * 2 + N_ROWS * 8 + N_ROWS * 8
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


def timed(fn, iters: int, warmup: int = 5) -> float:
    """Mean seconds per call over `iters` calls between two CUDA events (after `warmup` untimed calls)."""
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


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("calibration_times.py measures the GPU: no CUDA device")
    from metrics_b200.classification import MulticlassCalibrationError
    from metrics_b200.functional.classification.calibration_error import _ce_compute
    from oracle import calibration as oc

    dev = torch.device("cuda:0")
    info = card()
    g = torch.Generator().manual_seed(0)
    logits = torch.randn(N_ROWS, N_CLASSES, generator=g).bfloat16().to(dev)
    target = torch.randint(0, N_CLASSES, (N_ROWS,), generator=g).to(dev)

    metric = MulticlassCalibrationError(N_CLASSES, validate_args=False).to(dev)

    def update():
        metric.update(logits, target)
        metric.confidences.clear()
        metric.accuracies.clear()

    t_update = timed(update, args.iters)
    t_chain = timed(lambda: oc.multiclass_calibration_update_chain(logits, target, N_CLASSES), args.iters)
    metric.update(logits, target)
    conf, acc = metric.confidences[0], metric.accuracies[0]
    want_conf, want_acc = oc.multiclass_calibration_update_chain(logits, target, N_CLASSES)
    states_equal = bool(torch.equal(conf.view(torch.int32), want_conf.view(torch.int32)) and torch.equal(acc, want_acc))

    n = 10**7
    gc = torch.Generator(device=dev).manual_seed(1)
    big_conf = torch.rand(n, generator=gc, device=dev)
    big_acc = (torch.rand(n, generator=gc, device=dev) < big_conf).float()
    t_compute = timed(lambda: _ce_compute(big_conf, big_acc, 15, "l1"), max(5, args.iters // 5))
    t_compute_chain = timed(lambda: oc.ce_compute_chain(big_conf, big_acc, 15, "l1"), max(5, args.iters // 5))
    ece = float(_ce_compute(big_conf, big_acc, 15, "l1"))
    ece_chain = float(oc.ce_compute_chain(big_conf, big_acc, 15, "l1"))

    peak = PEAK_BW.get(info["name"])
    print(json.dumps({
        "card": info["name"], "power_limit_w": info["power_limit_w"],
        "update_us": round(t_update * 1e6, 2), "update_floor_bytes": FLOOR_BYTES,
        "update_achieved_tb_s": round(FLOOR_BYTES / t_update / 1e12, 3),
        "update_share_of_datasheet_bw": None if peak is None else round(FLOOR_BYTES / t_update / peak, 3),
        "chain_update_us": round(t_chain * 1e6, 2), "states_bit_equal_to_chain": states_equal,
        "compute_1e7_us": round(t_compute * 1e6, 2), "chain_compute_1e7_us": round(t_compute_chain * 1e6, 2),
        "compute_1e7_ece": ece, "chain_compute_1e7_ece": ece_chain, "compute_abs_diff": abs(ece - ece_chain),
        "iters": args.iters,
    }))


if __name__ == "__main__":
    main()
