"""CPU: the public surface, state registry and argument errors of the retrieval metrics against the reference's
(tests/golden/retrieval_surface.json, dumped by tests/golden/make_golden_retrieval.py).  Every error here is raised before
any kernel runs."""
import json
import os

import pytest
import torch

from tests.conftest import GOLDEN_DIR
from tests.golden.make_golden_retrieval import CLASSES, FUNCTIONALS, ret_states, ret_surface


@pytest.fixture(scope="module")
def ref():
    return json.load(open(os.path.join(GOLDEN_DIR, "retrieval_surface.json")))


def test_surface_matches_the_reference(ref):
    assert ret_surface("metrics_b200") == ref["surface"]


def test_state_registry_matches_the_reference(ref):
    assert ret_states("metrics_b200") == ref["states"]


def _calls():
    from metrics_b200 import retrieval as R  # noqa: N812
    from metrics_b200.functional import retrieval as F  # noqa: N812

    p4, t4, i4 = torch.rand(4), torch.tensor([0, 1, 0, 1]), torch.zeros(4, dtype=torch.long)
    calls = {}
    for cls in CLASSES:
        c = getattr(R, cls)
        calls[f"{cls}/empty_target_action"] = lambda c=c: c(empty_target_action="casual")
        calls[f"{cls}/ignore_index"] = lambda c=c: c(ignore_index=1.5)
        calls[f"{cls}/aggregation"] = lambda c=c: c(aggregation="sum")
        if cls != "RetrievalRPrecision":
            calls[f"{cls}/top_k_neg"] = lambda c=c: c(top_k=-1)
            calls[f"{cls}/top_k_float"] = lambda c=c: c(top_k=1.5)
            calls[f"{cls}/top_k_neg_float"] = lambda c=c: c(top_k=-1.5)
        calls[f"{cls}/indexes_none"] = lambda c=c: c().update(p4, t4, None)
        calls[f"{cls}/shape"] = lambda c=c: c().update(p4, t4[:3], i4)
        calls[f"{cls}/indexes_dtype"] = lambda c=c: c().update(p4, t4, i4.int())
        calls[f"{cls}/all_ignored"] = lambda c=c: c(ignore_index=1).update(p4[1::2], t4[1::2], i4[1::2])
        calls[f"{cls}/target_dtype"] = lambda c=c: c().update(p4, t4.to(torch.uint8), i4)
        calls[f"{cls}/preds_dtype"] = lambda c=c: c().update(t4, t4, i4)
        calls[f"{cls}/non_binary"] = lambda c=c: c().update(p4, t4 * 2, i4)
    calls["RetrievalPrecision/adaptive_k"] = lambda: R.RetrievalPrecision(adaptive_k=1)
    for fname in FUNCTIONALS:
        fn = getattr(F, fname)
        calls[f"{fname}/shape"] = lambda fn=fn: fn(p4, t4[:3])
        calls[f"{fname}/empty"] = lambda fn=fn: fn(p4[:0], t4[:0])
        calls[f"{fname}/scalar"] = lambda fn=fn: fn(p4[0], t4[0])
        calls[f"{fname}/non_binary"] = lambda fn=fn: fn(p4, t4 * 2)
        if fname != "retrieval_r_precision":
            calls[f"{fname}/top_k_zero"] = lambda fn=fn: fn(p4, t4, top_k=0)
            calls[f"{fname}/top_k_neg_float"] = lambda fn=fn: fn(p4, t4, top_k=-1.5)
    calls["retrieval_precision/adaptive_k"] = lambda: F.retrieval_precision(p4, t4, adaptive_k=1)
    calls["retrieval_r_precision/float_target"] = lambda: F.retrieval_r_precision(p4, t4.float())
    return calls


def test_argument_errors_match_the_reference(ref):
    errors = ref["errors"]
    for name, call in _calls().items():
        if name in errors:
            kind, msg = errors[name]
            with pytest.raises(Exception) as info:
                call()
            assert type(info.value).__name__ == kind and str(info.value) == msg, (name, info.value)
    # what the reference lets through (loose top_k checks, top_k=0 meaning "all" in AP / RR) is not rejected here either
    for name in ("RetrievalMAP/top_k_neg", "RetrievalMAP/top_k_float", "RetrievalMRR/top_k_neg", "RetrievalMRR/top_k_float"):
        assert name not in errors
        _calls()[name]()
    assert "RetrievalRPrecision/float_target" in errors  # raised at compute(): tests/test_retrieval_gpu.py


def test_not_exported_from_the_top_level_package():
    import metrics_b200

    assert not hasattr(metrics_b200, "RetrievalMAP")
