"""Generate tests/golden/rankcorr.npz from the UNMODIFIED reference (TorchMetrics under /root/reference), CPU tensors.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_rankcorr.py

Same import set-up as make_golden_retrieval.py.  Every case feeds one or more batches through a reference class
(`compute()`) and runs the functional on the concatenated batches.  Inputs are stored as float64 / int64 arrays with the
dtype name in the case's metadata (bfloat16 values are exact in float64).  The cases cover float16 / bfloat16 / float32 /
float64 for both metrics and int32 / int64 for Kendall; one and three outputs; continuous data, five tie levels, a constant
column, -0 / +0 and one NaN per column; N = 1 and N = 2; Kendall's variants a, b and c with the t-test under every
alternative.  Half-precision Spearman cases stay at N <= 256, where the reference's half-precision ranks are exact.
The reference's errors for invalid arguments and inputs are stored in the metadata as well.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
DTYPES = {"float16": torch.float16, "bfloat16": torch.bfloat16, "float32": torch.float32, "float64": torch.float64,
          "int32": torch.int32, "int64": torch.int64}


def _data(g, n, d, kind, dtype):
    """[n, d] (or [n] for d == 0) preds / target pair of the given kind."""
    dd = max(d, 1)
    x = torch.randn(n, dd, generator=g, dtype=torch.float64)
    y = 0.6 * x + 0.8 * torch.randn(n, dd, generator=g, dtype=torch.float64)
    if kind == "ties5" or not dtype.is_floating_point:
        scale = 1.0 if kind == "ties5" else 40.0
        x, y = (x * scale).round().clamp(-2 * scale, 2 * scale), (y * scale).round().clamp(-2 * scale, 2 * scale)
    if kind == "special" and n >= 4:
        x[:, 0] = 1.5  # a constant column
        y[: n // 2, -1] = 0.0
        y[n // 2:, -1] = -0.0 * y[n // 2:, -1].sign().abs()  # -0.0 mixed with +0.0
        y[n // 3:, -1] = y[n // 3:, -1].round()
        if dtype.is_floating_point:
            for c in range(dd):
                x[int(torch.randint(0, n, (1,), generator=g)), c] = float("nan")
                y[int(torch.randint(0, n, (1,), generator=g)), c] = float("nan")
    x, y = x.to(dtype), y.to(dtype)
    return (x[:, 0], y[:, 0]) if d == 0 else (x, y)


def _np(t):
    return t.double().numpy() if t.dtype.is_floating_point else t.long().numpy()


def rankcorr_golden():
    from torchmetrics.functional.regression import kendall_rank_corrcoef, spearman_corrcoef
    from torchmetrics.regression import KendallRankCorrCoef, SpearmanCorrCoef

    g = torch.Generator().manual_seed(1717)
    out, meta = {}, []

    def put(metric, dtype, kind, sizes, d, kwargs=None):
        kwargs = kwargs or {}
        key = f"case{len(meta)}"
        batches = [_data(g, n, d, kind, DTYPES[dtype]) for n in sizes]
        num_outputs = max(d, 1)
        if metric == "spearman":
            m = SpearmanCorrCoef(num_outputs=num_outputs)
        else:
            m = KendallRankCorrCoef(num_outputs=num_outputs, **kwargs)
        for b, (p, t) in enumerate(batches):
            m.update(p, t)
            out[f"{key}/preds{b}"], out[f"{key}/target{b}"] = _np(p), _np(t)
        res = m.compute()
        p = torch.cat([b[0] for b in batches])
        t = torch.cat([b[1] for b in batches])
        fres = spearman_corrcoef(p, t) if metric == "spearman" else kendall_rank_corrcoef(p, t, **kwargs)
        result_dtype = {}
        for name, r in (("compute", res), ("functional", fres)):
            if isinstance(r, tuple):
                out[f"{key}/{name}_p"] = r[1].double().numpy()
                r = r[0]
            out[f"{key}/{name}"] = r.double().numpy()
            result_dtype[name] = str(r.dtype).replace("torch.", "")
        meta.append({"metric": metric, "dtype": dtype, "kind": kind, "sizes": list(sizes), "d": d, "kwargs": kwargs,
                     "compute_dtype": result_dtype["compute"], "functional_dtype": result_dtype["functional"]})

    floats = ("float16", "bfloat16", "float32", "float64")
    for dtype in floats:
        small = dtype in ("float16", "bfloat16")
        for kind in ("cont", "ties5", "special"):
            put("spearman", dtype, kind, (60, 90, 100) if small else (400, 700), 0)
            put("spearman", dtype, kind, (120, 130) if small else (500, 300, 200), 3)
        put("spearman", dtype, "cont", (1,), 0)
        put("spearman", dtype, "cont", (2,), 0)
        put("spearman", dtype, "cont", (1, 1), 3)
    put("spearman", "float32", "cont", (5000,), 0)
    put("spearman", "float64", "ties5", (5000,), 0)

    variants = [{"variant": v} for v in ("a", "b", "c")]
    tests = [{"variant": v, "t_test": True, "alternative": a} for v in ("a", "b", "c")
             for a in ("two-sided", "less", "greater")]
    for dtype in (*floats, "int32", "int64"):
        kinds = ("cont", "ties5", "special") if dtype in floats else ("cont", "ties5")
        for kind in kinds:
            for kw in variants:
                put("kendall", dtype, kind, (150, 250), 0, kw)
            put("kendall", dtype, kind, (200, 100), 3, {"variant": "b", "t_test": True, "alternative": "two-sided"})
        put("kendall", dtype, "cont", (1,), 0, {"variant": "b", "t_test": True})
        put("kendall", dtype, "cont", (2,), 0, {"variant": "b", "t_test": True})
    for i, kw in enumerate(tests):
        put("kendall", ("float32", "float64", "int64")[i % 3], ("cont", "ties5", "special")[i % 3], (300, 200), 0, kw)
        put("kendall", "float32", "special", (150,), 3, kw)
    for kw in ({"variant": "b", "t_test": True}, {"variant": "c", "t_test": True, "alternative": "greater"}):
        put("kendall", "float32", "cont", (5000,), 0, kw)
        put("kendall", "float64", "ties5", (2500, 2500), 0, kw)
    put("kendall", "int32", "ties5", (1,), 3, {"variant": "a", "t_test": True})
    put("kendall", "int32", "ties5", (2,), 3, {"variant": "c", "t_test": True})

    # the reference's errors for invalid arguments and inputs
    errors = {}

    def err(name, fn):
        try:
            fn()
        except Exception as e:  # noqa: BLE001
            errors[name] = [type(e).__name__, str(e)]

    p4, t4 = torch.rand(4), torch.rand(4)
    err("spearman/int_inputs", lambda: spearman_corrcoef(torch.arange(4), torch.arange(4)))
    err("spearman/shape", lambda: spearman_corrcoef(p4, t4[:3]))
    err("spearman/ndim", lambda: spearman_corrcoef(torch.rand(4, 2, 2), torch.rand(4, 2, 2)))
    err("SpearmanCorrCoef/num_outputs", lambda: SpearmanCorrCoef(num_outputs=2).update(torch.rand(4, 3), torch.rand(4, 3)))
    err("SpearmanCorrCoef/one_output_2d", lambda: SpearmanCorrCoef().update(torch.rand(4, 3), torch.rand(4, 3)))
    err("kendall/shape", lambda: kendall_rank_corrcoef(p4, t4[:3]))
    err("kendall/ndim", lambda: kendall_rank_corrcoef(torch.rand(4, 2, 2), torch.rand(4, 2, 2)))
    err("kendall/variant", lambda: kendall_rank_corrcoef(p4, t4, variant="d"))
    err("kendall/alternative", lambda: kendall_rank_corrcoef(p4, t4, t_test=True, alternative="both"))
    err("kendall/t_test", lambda: kendall_rank_corrcoef(p4, t4, t_test=1))
    err("kendall/alternative_none", lambda: kendall_rank_corrcoef(p4, t4, t_test=True, alternative=None))
    err("KendallRankCorrCoef/variant", lambda: KendallRankCorrCoef(variant="x"))
    err("KendallRankCorrCoef/t_test", lambda: KendallRankCorrCoef(t_test="yes"))
    err("KendallRankCorrCoef/alternative_none", lambda: KendallRankCorrCoef(t_test=True, alternative=None))
    err("KendallRankCorrCoef/alternative", lambda: KendallRankCorrCoef(t_test=True, alternative="more"))
    err("KendallRankCorrCoef/num_outputs", lambda: KendallRankCorrCoef(num_outputs=2).update(torch.rand(4, 3), torch.rand(4, 3)))
    return out, meta, errors


if __name__ == "__main__":
    import warnings

    warnings.simplefilter("ignore")
    sys.path.insert(0, os.path.join(HERE, "_standins"))
    sys.path.insert(0, "/root/reference/src")
    data, meta, errors = rankcorr_golden()
    data["meta"] = np.array(json.dumps(meta))
    data["errors"] = np.array(json.dumps(errors))
    path = os.path.join(HERE, "rankcorr.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB,", len(meta), "cases,", len(errors), "errors")
