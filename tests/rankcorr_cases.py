"""Shared helpers of the rank-correlation tests: the goldens of tests/golden/rankcorr.npz (written from the unmodified
reference by make_golden_rankcorr.py), their inputs as tensors, and the tolerance each case is held to."""
import json
import os

import numpy as np
import torch

from tests.conftest import GOLDEN_DIR

DTYPES = {"float16": torch.float16, "bfloat16": torch.bfloat16, "float32": torch.float32, "float64": torch.float64,
          "int32": torch.int32, "int64": torch.int64}


def load():
    return np.load(os.path.join(GOLDEN_DIR, "rankcorr.npz"), allow_pickle=False)


def cases(golden):
    return [(f"case{i}", m) for i, m in enumerate(json.loads(str(golden["meta"])))]


def errors(golden) -> dict:
    return json.loads(str(golden["errors"]))


def batches(golden, key, meta, device="cpu"):
    dt = DTYPES[meta["dtype"]]
    return [(torch.from_numpy(golden[f"{key}/preds{b}"]).to(dt).to(device),
             torch.from_numpy(golden[f"{key}/target{b}"]).to(dt).to(device)) for b in range(len(meta["sizes"]))]


def several_nans_per_column(meta) -> bool:
    """The reference orders several NaNs of one column by an unstable argsort; K17 keeps their arrival order (deviation)."""
    return meta["kind"] == "special" and len(meta["sizes"]) > 1 and meta["dtype"].startswith(("float", "bfloat"))


def spacing(v, dtype: str) -> np.ndarray:
    """One unit in the last place of |v| in `dtype` (at least that of 2^-10, so values near 0 keep a usable scale)."""
    v = np.maximum(np.abs(np.asarray(v, np.float64)), 2.0 ** -10)
    if dtype == "bfloat16":
        return 2.0 ** (np.floor(np.log2(v)) - 7)
    return np.spacing(v.astype({"float16": np.float16, "float32": np.float32, "float64": np.float64}[dtype])).astype(np.float64)


def ulp_close(got, want, dtype: str, ulps: float) -> bool:
    got, want = np.atleast_1d(np.asarray(got, np.float64)), np.atleast_1d(np.asarray(want, np.float64))
    if got.shape != want.shape or not np.array_equal(np.isnan(got), np.isnan(want)):
        return False
    ok = ~np.isnan(want)
    return bool(np.all(np.abs(got[ok] - want[ok]) <= ulps * spacing(want[ok], dtype)))


def spearman_ulps(dtype: str) -> float:
    """Spearman against the reference: the reference ranks, averages and multiplies in the input dtype, so its float32
    result carries a few float32 roundings and its float16 / bfloat16 result a few half-precision ones; float64 agrees to
    2 ulp."""
    return {"float64": 2, "float32": 4}.get(dtype, 3)


def half_overflow(meta) -> bool:
    """Kendall variant c on float16 inputs: the reference computes n^2 in float16, which overflows past 255 rows and turns
    tau into 0 or NaN (deviation: K17 computes it exactly)."""
    return meta["metric"] == "kendall" and meta["functional_dtype"] == "float16" and sum(meta["sizes"]) ** 2 > 65504
