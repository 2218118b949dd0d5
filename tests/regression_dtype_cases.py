"""Replay of tests/golden/regression_dtypes.npz (tests/golden/make_golden_regression_dtypes.py): the regression functionals
on mixed-dtype pairs, N-d inputs and a `num_outputs` that is not the row width, against the reference's values.  Used by the
CPU suite (kernel stand-ins) and the GPU suite (the kernel)."""
import json

import numpy as np
import torch

DTYPES = {0: torch.float32, 1: torch.float16, 2: torch.bfloat16, 3: torch.float64}


def replay(g, dev: str) -> int:
    import metrics_b200.functional.regression as F

    n = int(g["n_cases"])
    for c in range(n):
        key = f"case{c}"
        fn, kwargs = str(g[f"{key}/fn"]), json.loads(str(g[f"{key}/kwargs"]))
        dp, dt, dv = (DTYPES[int(x)] for x in g[f"{key}/dtypes"])
        preds = torch.from_numpy(g[f"{key}/preds"]).to(dp).to(dev)
        target = torch.from_numpy(g[f"{key}/target"]).to(dt).to(dev)
        got = getattr(F, fn)(preds, target, **kwargs)
        want = g[f"{key}/value_promoted"]  # the terms are computed in the promoted dtype (DESIGN, K9)
        msg = f"{key}: {fn}({dp}, {dt}, {kwargs})"
        assert got.dtype == dv, f"{msg}: dtype {got.dtype}, reference {dv}"
        assert tuple(got.shape) == want.shape, f"{msg}: shape {tuple(got.shape)}, reference {want.shape}"
        # float64 results: the reference computes in float64 too.  float32: the reference's float32 `torch.sum` and, for
        # R2 / explained variance / RSE, its difference of nearly equal float32 sums.
        tol = dict(rtol=1e-10, atol=1e-12) if dv == torch.float64 else dict(rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(got.double().cpu().numpy(), want, err_msg=msg, **tol)
    return n
