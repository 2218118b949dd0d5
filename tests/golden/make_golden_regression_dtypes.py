"""Generate tests/golden/regression_dtypes.npz from the UNMODIFIED reference (TorchMetrics under /root/reference), CPU tensors.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_regression_dtypes.py

Same import set-up as make_golden.py.  The cases are the regression functionals on inputs whose dtypes differ (the
reference promotes them), on N-d inputs whose dims past the first are all kept by a dim-0 reduction, and a `num_outputs`
that does not divide the row width.  Every case stores its inputs, the functional and its keyword arguments, the
reference's value with its dtype, and the reference's value on both inputs cast to the promoted dtype first
(tests/regression_dtype_cases.py replays them).
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "_standins"))
sys.path.insert(0, "/root/reference/src")

import torchmetrics.functional.regression as R  # noqa: E402

DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2, torch.float64: 3}


def np_of(t: torch.Tensor) -> np.ndarray:
    """float16 / bfloat16 are stored widened to float32 (exact); the dtype code says what to narrow them back to."""
    return t.float().numpy() if t.dtype in (torch.float16, torch.bfloat16) else t.numpy()


def regression_dtypes_golden() -> dict:
    g = torch.Generator().manual_seed(909)
    out = {}
    case = 0

    def put(fn, preds, target, **kwargs):
        nonlocal case
        key = f"case{case}"
        value = getattr(R, fn)(preds, target, **kwargs)
        out[f"{key}/fn"] = np.array(fn)
        out[f"{key}/kwargs"] = np.array(json.dumps(kwargs, sort_keys=True))
        out[f"{key}/preds"], out[f"{key}/target"] = np_of(preds), np_of(target)
        out[f"{key}/value"] = np_of(value)
        # the reference on both inputs cast to the promoted dtype first: it differs from `value` where the reference
        # evaluates part of its chain in an operand's own half-precision dtype (MSLE's log1p, Tweedie's pow, the
        # target-only sums of WMAPE / RSE), which the kernel does not do
        promoted = torch.promote_types(preds.dtype, target.dtype)
        out[f"{key}/value_promoted"] = np_of(getattr(R, fn)(preds.to(promoted), target.to(promoted), **kwargs))
        out[f"{key}/dtypes"] = np.array([DTYPE_CODE[preds.dtype], DTYPE_CODE[target.dtype], DTYPE_CODE[value.dtype]])
        case += 1

    # mixed dtypes: every functional, both operand orders, target = preds + small noise (computing in the narrower dtype
    # instead of the promoted one shows most when the two are close)
    pairs = [(torch.float16, torch.float32), (torch.float32, torch.float16), (torch.bfloat16, torch.float32),
             (torch.float32, torch.bfloat16), (torch.float32, torch.float64), (torch.float64, torch.float32)]
    for dp, dt in pairs:
        base = torch.randn(400, generator=g, dtype=torch.float64)
        noise = 1e-3 * torch.randn(400, generator=g, dtype=torch.float64)
        p, t = base.to(dp), (base + noise).to(dt)
        for fn in ("mean_squared_error", "mean_absolute_error", "mean_absolute_percentage_error",
                   "symmetric_mean_absolute_percentage_error", "weighted_mean_absolute_percentage_error", "r2_score",
                   "relative_squared_error", "explained_variance"):
            put(fn, p, t)
        put("mean_squared_error", p, t, squared=False)
        # the transcendental terms cancel when preds and target are close: keep them apart, so that the reference's float32
        # evaluation is not dominated by its own rounding
        far = (base + 300 * noise).to(dt)
        put("log_cosh_error", p, far)
        put("minkowski_distance", p, far, p=3)
        pos_p, pos_t = (base.abs() + 0.5).to(dp), ((base.abs() + 0.5) * torch.exp(300 * noise)).to(dt)
        put("mean_squared_log_error", pos_p, pos_t)
        for power in (0.0, 1.0, 1.5, 2.0, 3.0):
            put("tweedie_deviance_score", pos_p, pos_t, power=power)
        p2 = base.reshape(80, 5).to(dp)
        t2 = (base + noise).reshape(80, 5).to(dt)
        put("mean_squared_error", p2, t2, num_outputs=5)
        put("r2_score", p2, t2, multioutput="raw_values")
        put("explained_variance", p2, t2, multioutput="raw_values")

    # N-d inputs: every dim past the first is kept by the dim-0 reductions
    p, t = torch.randn(40, 3, 2, generator=g), torch.randn(40, 3, 2, generator=g)
    put("mean_squared_error", p, t, num_outputs=3)
    put("mean_squared_error", p, t, num_outputs=3, squared=False)
    put("mean_absolute_error", p, t, num_outputs=3)
    put("mean_squared_error", p, t)
    p, t = torch.randn(50, 3, 4, generator=g), torch.randn(50, 3, 4, generator=g)
    for mo in ("raw_values", "uniform_average", "variance_weighted"):
        put("explained_variance", p, t, multioutput=mo)
    put("explained_variance", p.double(), t.float(), multioutput="raw_values")
    # num_outputs that is not the row width: the reference still sums over dim 0
    p, t = torch.randn(10, 4, generator=g), torch.randn(10, 4, generator=g)
    put("mean_squared_error", p, t, num_outputs=3)
    put("mean_absolute_error", p, t, num_outputs=3)
    out["n_cases"] = np.array(case)
    return out


if __name__ == "__main__":
    data = regression_dtypes_golden()
    path = os.path.join(HERE, "regression_dtypes.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB,", len(data), "arrays")
