"""Kernel K17 (SpearmanCorrCoef, KendallRankCorrCoef): `compute()` time of both metrics and the time of one native call
(CUDA events) at N in {10^4, 10^6, 10^7} rows x D in {1, 8} outputs, for continuous data and for data with five tie levels;
the reference's algorithms restated as torch ops on the same GPU (oracle/rank_corr.py: torch_spearman_loop, one masked mean
per repeated value, up to 10^6 rows; torch_kendall_pairs_loop, one Python iteration per row, up to 2 * 10^4 rows).  Every
timed result is checked against the float64 oracle (column 0).  Prints one JSON line per workload as it finishes, then one
with the card name and power limit, read in the same run.
Usage: python benchmarks/rankcorr_times.py [--iters 5]
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

from benchmarks.retrieval_times import events, wall  # noqa: E402
from benchmarks.segmentation_times import card  # noqa: E402


def data(n, d, tied, dev):
    g = torch.Generator(device=dev).manual_seed(17)
    x = torch.randn(n, d, generator=g, device=dev)
    y = 0.6 * x + 0.8 * torch.randn(n, d, generator=g, device=dev)
    if tied:
        x, y = (x * 1.25).round().clamp(-2, 2), (y * 1.25).round().clamp(-2, 2)
    return x, y


def fresh_compute(m):
    m._computed = None
    return m.compute()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    from metrics_b200 import _native
    from metrics_b200.regression import KendallRankCorrCoef, SpearmanCorrCoef
    from oracle import rank_corr as orc

    dev = torch.device("cuda:0")
    c = card()
    out = {"card": c["name"], "power_limit_w": c["power_limit_w"], "iters": args.iters}
    for n in (10 ** 4, 10 ** 6, 10 ** 7):
        for d in (1, 8):
            for tied in (False, True):
                x, y = data(n, d, tied, dev)
                res = {}
                rho = SpearmanCorrCoef(num_outputs=d).to(dev)
                tau = KendallRankCorrCoef(num_outputs=d, t_test=True).to(dev)
                rho.update(x if d > 1 else x[:, 0], y if d > 1 else y[:, 0])
                tau.update(x if d > 1 else x[:, 0], y if d > 1 else y[:, 0])
                res["spearman_compute_ms"] = round(wall(lambda: fresh_compute(rho), args.iters) * 1e3, 3)
                res["kendall_compute_ms"] = round(wall(lambda: fresh_compute(tau), args.iters) * 1e3, 3)
                res["spearman_call_ms"] = round(events(lambda: _native.spearman_corrcoef(x, y, torch.float32), args.iters) * 1e3, 3)
                res["kendall_call_ms"] = round(events(lambda: _native.kendall_rank_corrcoef(x, y, "b", "two-sided"), args.iters) * 1e3, 3)
                x0, y0 = x[:, 0].double().cpu().numpy(), y[:, 0].double().cpu().numpy()
                got_rho = np.atleast_1d(fresh_compute(rho).cpu().numpy())[0]
                got_tau, got_p = (np.atleast_1d(v.cpu().numpy())[0] for v in fresh_compute(tau))
                want_tau, want_p = orc.kendall(x0, y0, "b", "two-sided")
                res["spearman_abs_diff_oracle"] = float(abs(got_rho - orc.spearman(x0, y0)[0]))
                res["kendall_tau_abs_diff_oracle"] = float(abs(got_tau - want_tau[0]))
                res["kendall_p_abs_diff_oracle"] = float(abs(got_p - want_p[0]))
                if n <= 10 ** 6:
                    res["torch_spearman_loop_ms"] = round(wall(lambda: orc.torch_spearman_loop(x, y), 1) * 1e3, 1)
                else:
                    res["torch_spearman_loop_ms"] = "not measured"
                if n <= 2 * 10 ** 4 and d == 1:
                    res["torch_kendall_pairs_loop_ms"] = round(wall(lambda: orc.torch_kendall_pairs_loop(x, y), 1) * 1e3, 1)
                    conc, disc = orc.torch_kendall_pairs_loop(x, y)
                    st = orc.kendall_stats(x0, y0)
                    res["kendall_pairs_equal_loop"] = bool(int(conc[0]) == st["conc"] and int(disc[0]) == st["disc"])
                else:
                    res["torch_kendall_pairs_loop_ms"] = "not measured"
                out[f"n{n}_d{d}_{'ties5' if tied else 'cont'}"] = res
                print(json.dumps({f"n{n}_d{d}_{'ties5' if tied else 'cont'}": res}), flush=True)
                del rho, tau, x, y
                torch.cuda.empty_cache()
    x, y = data(2 * 10 ** 4, 1, False, dev)
    out["n20000_d1_cont_torch_kendall_pairs_loop_ms"] = round(wall(lambda: orc.torch_kendall_pairs_loop(x, y), 1) * 1e3, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
