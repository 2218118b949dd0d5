"""The retrieval goldens (tests/golden/retrieval.npz, from tests/golden/make_golden_retrieval.py): loading, and one case
run through this package's class and functional, shared by the oracle and GPU tests."""
import json
import os

import numpy as np
import torch

from tests.conftest import GOLDEN_DIR

KIND = {"RetrievalMAP": "map", "RetrievalMRR": "mrr", "RetrievalPrecision": "precision", "RetrievalRecall": "recall",
        "RetrievalHitRate": "hit_rate", "RetrievalFallOut": "fall_out", "RetrievalRPrecision": "r_precision",
        "RetrievalNormalizedDCG": "ndcg"}
FUNCTIONAL = {"RetrievalMAP": "retrieval_average_precision", "RetrievalMRR": "retrieval_reciprocal_rank",
              "RetrievalPrecision": "retrieval_precision", "RetrievalRecall": "retrieval_recall",
              "RetrievalHitRate": "retrieval_hit_rate", "RetrievalFallOut": "retrieval_fall_out",
              "RetrievalRPrecision": "retrieval_r_precision", "RetrievalNormalizedDCG": "retrieval_normalized_dcg"}


def load():
    return np.load(os.path.join(GOLDEN_DIR, "retrieval.npz"))


def cases(golden):
    for c, meta in enumerate(json.loads(str(golden["meta"]))):
        yield f"case{c}", meta


def batches(golden, key, meta):
    return [(golden[f"{key}/indexes{b}"], golden[f"{key}/preds{b}"], golden[f"{key}/target{b}"]) for b in range(meta["batches"])]


def concat(golden, key, meta):
    bs = batches(golden, key, meta)
    idx, p, t = (np.concatenate([b[i] for b in bs]) for i in range(3))
    ii = meta["kwargs"].get("ignore_index")
    if ii is not None:
        keep = t != ii
        idx, p, t = idx[keep], p[keep], t[keep]
    return idx, p, t


def ulp_close(got, want, ndcg: bool) -> bool:
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    if ndcg:
        return bool(np.allclose(got, want, rtol=1e-5, atol=1e-7))
    return bool(np.all(np.abs(got - want) <= np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)))


def identity(values, dim=None):
    return values


def check_case(golden, key, meta, device):
    """The class (aggregated and per-query) and the functional (per query) against the reference's values."""
    from metrics_b200 import retrieval as R  # noqa: N812
    from metrics_b200.functional import retrieval as F  # noqa: N812

    ndcg = meta["cls"] == "RetrievalNormalizedDCG"
    m = getattr(R, meta["cls"])(aggregation=meta["aggregation"], **meta["kwargs"]).to(device)
    mv = getattr(R, meta["cls"])(aggregation=identity, **meta["kwargs"]).to(device)
    for i, p, t in batches(golden, key, meta):
        args = (torch.from_numpy(p).to(device), torch.from_numpy(t).to(device), torch.from_numpy(i).to(device))
        m.update(*args[:2], indexes=args[2])
        mv.update(*args[:2], indexes=args[2])
    if meta["error"]:
        try:
            m.compute()
        except ValueError as e:
            assert str(e) == meta["error"], (key, e)
        else:
            raise AssertionError(f"{key}: no error")
        return
    got = float(m.compute())
    want = float(golden[f"{key}/compute"])
    assert np.isclose(got, want, rtol=1e-5 if ndcg else 2e-7, atol=1e-7), (key, meta, got, want)
    assert ulp_close(mv.compute().cpu().numpy(), golden[f"{key}/values"], ndcg), (key, meta)
    idx, p, t = concat(golden, key, meta)
    fkw = {k: v for k, v in meta["kwargs"].items() if k in ("top_k", "adaptive_k")}
    fn = getattr(F, FUNCTIONAL[meta["cls"]])
    wants = [v for v in golden[f"{key}/functional"] if not np.isnan(v)]  # queries whose records were all ignored
    for q, want_q in zip(np.unique(idx), wants):
        sel = idx == q
        got_q = float(fn(torch.from_numpy(p[sel]).to(device), torch.from_numpy(t[sel]).to(device), **fkw))
        assert ulp_close(got_q, want_q, ndcg), (key, q, got_q, want_q)
