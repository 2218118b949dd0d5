"""The goldens of RetrievalAUROC, RetrievalPrecisionRecallCurve and RetrievalRecallAtFixedPrecision
(tests/golden/retrieval_curves.npz, from tests/golden/make_golden_retrieval_curves.py): loading, and one case run through
this package's class and functional, shared by the oracle and GPU tests."""
import json
import os

import numpy as np
import torch

from tests.conftest import GOLDEN_DIR
from tests.retrieval_cases import batches, concat, identity

FUNCTIONAL = {"RetrievalAUROC": "retrieval_auroc", "RetrievalPrecisionRecallCurve": "retrieval_precision_recall_curve",
              "RetrievalRecallAtFixedPrecision": "retrieval_precision_recall_curve"}
# AUROC here is the correctly rounded float32 of an exact area; the reference's is a float32 trapezoid
AUROC_TOL = dict(rtol=1e-5, atol=1e-6, equal_nan=True)
# aggregated curves: float32 means over the queries, reduced in another order than on the CPU
MEAN_TOL = dict(rtol=1e-6, atol=1e-7)


def load():
    return np.load(os.path.join(GOLDEN_DIR, "retrieval_curves.npz"))


def cases(golden):
    for c, meta in enumerate(json.loads(str(golden["meta"]))):
        yield f"case{c}", meta


def integer_target(golden, key, meta) -> bool:
    return not np.issubdtype(golden[f"{key}/target0"].dtype, np.floating)


def curve_equal(got, want, exact: bool) -> bool:
    got, want = np.asarray(got, dtype=np.float32), np.asarray(want, dtype=np.float32)
    if got.shape != want.shape:
        return False
    return bool(np.array_equal(got, want)) if exact else bool(np.allclose(got, want, rtol=1e-6, atol=1e-7))


def _kwargs(meta):
    agg = meta["aggregation"]
    if meta["cls"] == "RetrievalRecallAtFixedPrecision" and agg == "mean":
        return dict(meta["kwargs"])
    return dict(meta["kwargs"], aggregation=agg)


def check_case(golden, key, meta, device):
    """The class (aggregated and per-query) and the functional (per query) against the reference's values."""
    from metrics_b200 import retrieval as R  # noqa: N812
    from metrics_b200.functional import retrieval as F  # noqa: N812

    cls = meta["cls"]
    exact = integer_target(golden, key, meta)
    m = getattr(R, cls)(**_kwargs(meta)).to(device)
    mv = getattr(R, cls)(**dict(meta["kwargs"], aggregation=identity)).to(device) if cls != "RetrievalRecallAtFixedPrecision" else None
    for i, p, t in batches(golden, key, meta):
        args = (torch.from_numpy(p).to(device), torch.from_numpy(t).to(device), torch.from_numpy(i).to(device))
        for x in (m, mv):
            if x is not None:
                x.update(*args[:2], indexes=args[2])
    if meta["error"]:
        kind, msg = meta["error"].split(": ", 1)
        if kind == "IndexError":  # max_fpr past the curve: ValueError here
            kind, msg = "ValueError", "`max_fpr` must be"
        try:
            m.compute()
        except ValueError as e:
            assert kind == "ValueError" and str(e).startswith(msg), (key, e)
        else:
            raise AssertionError(f"{key}: no error")
    elif cls == "RetrievalAUROC":
        assert np.allclose(float(m.compute()), float(golden[f"{key}/compute"]), **AUROC_TOL), (key, meta)
        assert np.allclose(mv.compute().cpu().numpy(), golden[f"{key}/values"], **AUROC_TOL), (key, meta)
    elif cls == "RetrievalPrecisionRecallCurve":
        prec, rec, top_k = m.compute()
        tol = MEAN_TOL if meta["aggregation"] == "mean" else dict(rtol=0, atol=0)
        assert np.allclose(prec.cpu().numpy(), golden[f"{key}/compute_precision"], **tol), (key, meta)
        assert np.allclose(rec.cpu().numpy(), golden[f"{key}/compute_recall"], **tol), (key, meta)
        assert np.array_equal(top_k.cpu().numpy(), golden[f"{key}/compute_top_k"]) and top_k.dtype == torch.int64
        pv, rv, _ = mv.compute()  # [Q', max_k]; zeros(max_k) when every query is skipped
        assert curve_equal(np.atleast_2d(pv.cpu().numpy()), golden[f"{key}/values_precision"], exact), (key, meta)
        assert curve_equal(np.atleast_2d(rv.cpu().numpy()), golden[f"{key}/values_recall"], exact), (key, meta)
    else:
        r, k = m.compute()
        assert r.device.type == k.device.type == torch.device(device).type and r.dtype == torch.float32 and k.dtype == torch.int64
        assert np.isclose(float(r), float(golden[f"{key}/compute_recall"]), **MEAN_TOL), (key, meta, float(r))
        assert int(k) == int(golden[f"{key}/compute_k"]), (key, meta, int(k))
    if meta["functional_error"]:
        return
    idx, p, t = concat(golden, key, meta)
    fn = getattr(F, FUNCTIONAL[cls])
    fkw = {k: v for k, v in meta["kwargs"].items() if k in ("top_k", "max_fpr", "max_k", "adaptive_k")}
    queries = np.unique(idx)
    if cls == "RetrievalAUROC":
        got = [float(fn(torch.from_numpy(p[idx == q]).to(device), torch.from_numpy(t[idx == q]).to(device), **fkw)) for q in queries]
        assert np.allclose(got, golden[f"{key}/functional"], **AUROC_TOL), (key, meta)
        return
    bounds = np.concatenate([[0], np.cumsum(golden[f"{key}/functional_len"])])
    for j, q in enumerate(queries):
        pr, rc, tk = fn(torch.from_numpy(p[idx == q]).to(device), torch.from_numpy(t[idx == q]).to(device), **fkw)
        s = slice(bounds[j], bounds[j + 1])
        assert curve_equal(pr.cpu().numpy(), golden[f"{key}/functional_precision"][s], exact), (key, q)
        assert curve_equal(rc.cpu().numpy(), golden[f"{key}/functional_recall"][s], exact), (key, q)
        assert np.array_equal(tk.cpu().numpy(), golden[f"{key}/functional_top_k"][s]), (key, q)
