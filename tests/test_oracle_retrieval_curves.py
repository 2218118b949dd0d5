"""CPU: the float64 oracle of RetrievalAUROC, RetrievalPrecisionRecallCurve and RetrievalRecallAtFixedPrecision
(oracle/retrieval_curves.py) against every golden of the unmodified reference (tests/golden/retrieval_curves.npz)."""
import numpy as np
import pytest

from oracle import retrieval_curves as orc
from tests import retrieval_curves_cases as rcc
from tests.retrieval_cases import concat


def _oracle_compute(meta, idx, p, t):
    kw, agg = meta["kwargs"], meta["aggregation"]
    action = kw.get("empty_target_action", "neg")
    if meta["cls"] == "RetrievalAUROC":
        return orc.compute_auroc(idx, p, t, kw.get("top_k"), kw.get("max_fpr"), action, agg)
    curve = orc.compute_pr_curve(idx, p, t, kw.get("max_k"), kw.get("adaptive_k", False), action, agg)
    if meta["cls"] == "RetrievalPrecisionRecallCurve":
        return curve
    return orc.recall_at_fixed_precision(curve[0].astype(np.float32), curve[1].astype(np.float32), kw.get("min_precision", 0.0))


def test_oracle_against_every_golden():
    golden = rcc.load()
    for key, meta in rcc.cases(golden):
        idx, p, t = concat(golden, key, meta)
        kw = meta["kwargs"]
        if meta["error"]:
            with pytest.raises((ValueError, IndexError)):
                _oracle_compute(meta, idx, p, t)
            continue
        got = _oracle_compute(meta, idx, p, t)
        if meta["cls"] == "RetrievalAUROC":
            assert np.allclose(got, float(golden[f"{key}/compute"]), **rcc.AUROC_TOL), (key, meta)
            fvals = [orc.query_auroc(pq, tq, kw.get("top_k"), kw.get("max_fpr")) for _, pq, tq in orc.groups(idx, p, t)]
            assert np.allclose(fvals, golden[f"{key}/functional"], **rcc.AUROC_TOL), (key, meta)
        elif meta["cls"] == "RetrievalPrecisionRecallCurve":
            assert np.allclose(got[0], golden[f"{key}/compute_precision"], **rcc.MEAN_TOL), (key, meta)
            assert np.allclose(got[1], golden[f"{key}/compute_recall"], **rcc.MEAN_TOL), (key, meta)
            prec, rec, empty = orc.per_query_pr_curve(idx, p, t, kw.get("max_k"), kw.get("adaptive_k", False))
            action = kw.get("empty_target_action", "neg")
            prec, rec = orc._apply_action(prec, empty, action), orc._apply_action(rec, empty, action)
            exact = rcc.integer_target(golden, key, meta)
            if len(prec):
                assert rcc.curve_equal(prec, golden[f"{key}/values_precision"], exact), (key, meta)
                assert rcc.curve_equal(rec, golden[f"{key}/values_recall"], exact), (key, meta)
        else:
            assert np.isclose(got[0], float(golden[f"{key}/compute_recall"]), **rcc.MEAN_TOL), (key, meta, got)
            assert got[1] == int(golden[f"{key}/compute_k"]), (key, meta, got)


def test_sigmoid_ties_and_partial_area_by_hand():
    # 17, 18 and 25 all have the float32 probability 1.0: one tie group holding two positives and a negative
    assert orc.query_auroc(np.array([17.0, 18.0, 25.0, -3.0]), np.array([0, 1, 1, 0])) == 0.75
    # without logits the same order is strict and separates the classes
    assert orc.query_auroc(np.array([.17, .18, .25, .03]), np.array([0, 1, 1, 0])) == 1.0
    assert np.isnan(orc.query_auroc(np.array([.9, .1, .5]), np.array([1, 0, 0]), max_fpr=0.0))
    assert orc.recall_at_fixed_precision([1.0, .5, .5], [.5, 1.0, 1.0], 0.5) == (1.0, 3)
    assert orc.recall_at_fixed_precision([0.1, .2], [.5, 1.0], 0.5) == (0.0, 2)
