"""Kernels K16e / K16f (retrieval AUROC and precision-recall curve): `compute()` time of RetrievalAUROC(),
RetrievalAUROC(max_fpr=0.1), RetrievalPrecisionRecallCurve(max_k=100) and RetrievalRecallAtFixedPrecision(0.5, max_k=100),
the GPU time of each new entry point from CUDA events, and the reference's per-query loops restated with torch ops on the
same GPU (oracle/retrieval_curves.py: torch_loop_auroc, torch_loop_pr_curve) for u1e4 and r7k.

Workloads as in benchmarks/retrieval_times.py: u1e4 (10^4 queries x 100), r7k (7 000 x 1 000), pow (power-law lengths,
about 10^7 records), one (one query of 10^7).  Algorithmic bytes of an entry point: the sorted records read once (u64 key,
float32 target, 12 bytes each), plus 2 * Q * max_k * 4 bytes written for the curve.  Prints one JSON line with the card
name and power limit, read in the same run.  Usage: python benchmarks/retrieval_curves_times.py [--iters 5]
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

from benchmarks.retrieval_times import events, fresh_compute, wall, workload  # noqa: E402
from benchmarks.segmentation_times import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    from metrics_b200 import _native
    from metrics_b200.retrieval import RetrievalAUROC, RetrievalPrecisionRecallCurve, RetrievalRecallAtFixedPrecision
    from oracle.retrieval_curves import torch_loop_auroc, torch_loop_pr_curve

    dev = torch.device("cuda:0")
    c = card()
    out = {"card": c["name"], "power_limit_w": c["power_limit_w"], "iters": args.iters}
    for name in ("u1e4", "r7k", "pow", "one"):
        idx, p, t = workload(name, dev)
        n = idx.numel()
        res = {"n": n}
        for label, make in (("auroc", RetrievalAUROC), ("auroc_fpr01", lambda: RetrievalAUROC(max_fpr=0.1)),
                            ("prcurve100", lambda: RetrievalPrecisionRecallCurve(max_k=100)),
                            ("rafp05_100", lambda: RetrievalRecallAtFixedPrecision(0.5, max_k=100))):
            m = make().to(dev)
            m.update(p, t, indexes=idx)
            res[f"compute_{label}_ms"] = round(wall(lambda m=m: fresh_compute(m), args.iters) * 1e3, 3)
        groups = _native.retrieval_sort(idx, p, t)
        q = groups.num_queries
        res["queries"] = q
        res["auroc_kernel_ms"] = round(events(lambda: _native.retrieval_auroc(groups), args.iters) * 1e3, 3)
        res["auroc_fpr01_kernel_ms"] = round(events(lambda: _native.retrieval_auroc(groups, None, 0.1), args.iters) * 1e3, 3)
        res["prcurve100_kernel_ms"] = round(events(lambda: _native.retrieval_pr_curve(groups, 100), args.iters) * 1e3, 3)
        read, curve = n * 12, 2 * q * 100 * 4
        res["auroc_bytes"], res["prcurve100_bytes"] = read, read + curve
        res["auroc_gb_s"] = round(read / (res["auroc_kernel_ms"] / 1e3) / 1e9, 1)
        res["prcurve100_gb_s"] = round((read + curve) / (res["prcurve100_kernel_ms"] / 1e3) / 1e9, 1)
        if name in ("u1e4", "r7k"):
            res["torch_loop_auroc_ms"] = round(wall(lambda: torch_loop_auroc(idx, p, t), 1) * 1e3, 1)
            res["torch_loop_prcurve100_ms"] = round(wall(lambda: torch_loop_pr_curve(idx, p, t, 100), 1) * 1e3, 1)
            got = _native.retrieval_auroc(groups)[0].cpu().numpy()
            want = torch_loop_auroc(idx, p, t).cpu().numpy()
            res["auroc_max_abs_diff_baseline"] = float(np.abs(got.astype(np.float64) - want).max())
            res["auroc_values_equal_baseline"] = bool(np.allclose(got, want, rtol=1e-5, atol=1e-6))
            gp, gr, _ = (x.cpu().numpy() for x in _native.retrieval_pr_curve(groups, 100))
            wp, wr = (x.cpu().numpy() for x in torch_loop_pr_curve(idx, p, t, 100))
            res["prcurve_values_equal_baseline"] = bool(np.array_equal(gp, wp) and np.array_equal(gr, wr))
        else:
            res["torch_loop_auroc_ms"] = res["torch_loop_prcurve100_ms"] = "not measured"
        out[name] = res
        del groups
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
