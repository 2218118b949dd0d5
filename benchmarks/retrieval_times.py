"""Kernel K16 (retrieval): `compute()` time per metric and for a MAP + MRR + Precision@10 collection, the GPU time of the
group sort and of one evaluation, against the reference's per-query loop restated with torch ops on the same GPU
(oracle/retrieval.py: torch_loop).

  u1e4   10^4 queries x 100 documents          u1e5   10^5 queries x 100 documents
  r7k    7 000 queries x 1 000 documents       pow    power-law query lengths, about 10^7 records
  one    one query of 10^7 documents
Scores uniform, targets Bernoulli(0.1), records shuffled across queries.  Algorithmic bytes: the records read once (int64
index, float32 score, int64 target) and written once in sorted order (u64 key, float32 target), plus one read of the sorted
records by the evaluation.  Prints one JSON line with the card name and power limit, read in the same run.  Usage:
python benchmarks/retrieval_times.py [--iters 5]
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

from benchmarks.segmentation_times import card  # noqa: E402


def workload(name, dev):
    g = torch.Generator(device=dev).manual_seed(16)
    if name == "pow":
        gc = torch.Generator().manual_seed(16)
        lengths = (torch.rand(200_000, generator=gc) ** -1.2 * 8).long().clamp(max=200_000)
        lengths = lengths[: int((lengths.cumsum(0) < 10_000_000).sum())]
        idx = torch.repeat_interleave(torch.arange(len(lengths)), lengths).to(dev)
    else:
        q, d = {"u1e4": (10_000, 100), "u1e5": (100_000, 100), "r7k": (7_000, 1_000), "one": (1, 10_000_000)}[name]
        idx = torch.arange(q, device=dev).repeat_interleave(d)
    n = idx.numel()
    perm = torch.randperm(n, generator=g, device=dev)
    return idx[perm], torch.rand(n, generator=g, device=dev), (torch.rand(n, generator=g, device=dev) < 0.1).long()


def wall(fn, iters):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters


def events(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3 / iters


def fresh_compute(m):
    m._computed = None
    m._group_cache.clear()
    return m.compute()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    from metrics_b200 import _native
    from metrics_b200.collections import MetricCollection
    from metrics_b200.retrieval import RetrievalMAP, RetrievalMRR, RetrievalNormalizedDCG, RetrievalPrecision
    from oracle.retrieval import torch_loop

    dev = torch.device("cuda:0")
    c = card()
    out = {"card": c["name"], "power_limit_w": c["power_limit_w"], "iters": args.iters}
    for name in ("u1e4", "u1e5", "r7k", "pow", "one"):
        idx, p, t = workload(name, dev)
        n = idx.numel()
        res = {"n": n}
        for label, cls, kw in (("map", RetrievalMAP, {}), ("mrr", RetrievalMRR, {}), ("ndcg10", RetrievalNormalizedDCG, {"top_k": 10})):
            m = cls(**kw).to(dev)
            m.update(p, t, indexes=idx)
            res[f"compute_{label}_ms"] = round(wall(lambda m=m: fresh_compute(m), args.iters) * 1e3, 3)
        coll = MetricCollection({"map": RetrievalMAP(), "mrr": RetrievalMRR(), "p10": RetrievalPrecision(top_k=10)}).to(dev)
        coll.update(p, t, indexes=idx)

        def coll_compute():
            for m in coll.values():
                m._computed = None
                m._group_cache.clear()
            return coll.compute()

        res["compute_collection3_ms"] = round(wall(coll_compute, args.iters) * 1e3, 3)
        groups = _native.retrieval_sort(idx, p, t)
        res["queries"] = groups.num_queries
        res["sort_ms_incl_host_reads"] = round(wall(lambda: _native.retrieval_sort(idx, p, t), args.iters) * 1e3, 3)
        res["eval_map_kernel_ms"] = round(events(lambda: _native.retrieval_evaluate(groups, _native.RET_AP), args.iters) * 1e3, 3)
        algo = n * (8 + 4 + 8) + n * (8 + 4) + n * (8 + 4)
        res["algorithmic_bytes"] = algo
        res["achieved_gb_s"] = round(algo / ((res["sort_ms_incl_host_reads"] + res["eval_map_kernel_ms"]) / 1e3) / 1e9, 1)
        if name in ("u1e4", "r7k"):
            base = wall(lambda: torch_loop("map", idx, p, t), 1)
            res["torch_loop_map_ms"] = round(base * 1e3, 1)
            want = torch_loop("map", idx, p, t).cpu().numpy()
            got = _native.retrieval_evaluate(groups, _native.RET_AP)[0].cpu().numpy()
            res["values_equal_baseline"] = bool(np.array_equal(got, want))
            res["max_abs_diff_baseline"] = float(np.abs(got.astype(np.float64) - want).max())
        else:
            res["torch_loop_map_ms"] = "not measured"
        out[name] = res
        del groups
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
