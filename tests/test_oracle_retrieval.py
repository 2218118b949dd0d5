"""CPU: the retrieval oracle (oracle/retrieval.py) — the numpy float64 formulas and the torch restatement of the
reference's loop — reproduces every golden of tests/golden/retrieval.npz (dumped from the unmodified reference)."""
import numpy as np
import pytest
import torch

from oracle import retrieval as orc
from tests import retrieval_cases as rc


@pytest.fixture(scope="module")
def golden():
    return rc.load()


def _args(meta):
    kw = meta["kwargs"]
    return rc.KIND[meta["cls"]], kw.get("top_k"), kw.get("adaptive_k", False)


def test_oracle_reproduces_every_golden(golden):
    n = 0
    for key, meta in rc.cases(golden):
        if meta["stable_ties"]:
            continue
        kind, top_k, adaptive_k = _args(meta)
        idx, p, t = rc.concat(golden, key, meta)
        vals, empty = orc.per_query(kind, idx, p, t, top_k, adaptive_k)
        wants = [v for v in golden[f"{key}/functional"] if not np.isnan(v)]
        assert rc.ulp_close(vals.astype(np.float32), wants, kind == "ndcg"), (key, meta)
        action = meta["kwargs"].get("empty_target_action")
        if meta["error"]:
            with pytest.raises(ValueError):
                orc.compute(kind, idx, p, t, top_k, adaptive_k, action, meta["aggregation"])
            continue
        got = orc.compute(kind, idx, p, t, top_k, adaptive_k, action, meta["aggregation"])
        assert np.isclose(got, float(golden[f"{key}/compute"]), rtol=1e-5 if kind == "ndcg" else 2e-7, atol=1e-7), key
        n += 1
    assert n > 100


def test_torch_loop_reproduces_every_golden(golden):
    for key, meta in rc.cases(golden):
        if meta["stable_ties"]:
            continue
        kind, top_k, adaptive_k = _args(meta)
        idx, p, t = rc.concat(golden, key, meta)
        got = orc.torch_loop(kind, torch.from_numpy(idx), torch.from_numpy(p), torch.from_numpy(t), top_k, adaptive_k)
        wants = [v for v in golden[f"{key}/functional"] if not np.isnan(v)]
        assert rc.ulp_close(got.numpy(), wants, kind == "ndcg"), (key, meta)


def test_stable_tie_rule():
    p, t = np.array([.5, .5, .5, .1], np.float32), np.array([0, 1, 0, 1])
    assert orc.query_value("map", p, t) == 0.5
    assert float(orc.torch_loop("map", torch.zeros(4, dtype=torch.long), torch.from_numpy(p), torch.from_numpy(t))) == 0.5


def test_nan_rules():
    # outside NDCG a NaN score ranks first; in NDCG every NaN is its own tie group after all numbers, in input order
    p, t = np.array([0.2, np.nan, 0.9], np.float32), np.array([0, 1, 0])
    assert orc.query_value("mrr", p, t) == 1.0
    d = 1 / np.log2(np.arange(3) + 2)
    assert np.isclose(orc.query_value("ndcg", p, t), d[2] / d[0])
