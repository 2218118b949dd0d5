"""CPU: the public surface, state registry and argument errors of RetrievalAUROC, RetrievalPrecisionRecallCurve,
RetrievalRecallAtFixedPrecision and their functionals against the reference's (tests/golden/retrieval_curves_surface.json,
dumped by tests/golden/make_golden_retrieval_curves.py); the argument checks of the two C entry points, which fail
before any launch."""
import json
import os

import pytest
import torch

from tests.conftest import GOLDEN_DIR
from tests.golden.make_golden_retrieval_curves import (
    CLASSES,
    FUNCTIONALS,
    curves_states,
    curves_surface,
    error_calls_class,
    error_calls_functional,
)


@pytest.fixture(scope="module")
def ref():
    return json.load(open(os.path.join(GOLDEN_DIR, "retrieval_curves_surface.json")))


def test_surface_matches_the_reference(ref):
    assert curves_surface("metrics_b200") == ref["surface"]


def test_state_registry_matches_the_reference(ref):
    assert curves_states("metrics_b200") == ref["states"]


def _calls():
    from metrics_b200 import retrieval as R  # noqa: N812
    from metrics_b200.functional import retrieval as F  # noqa: N812

    p4, t4, i4 = torch.rand(4), torch.tensor([0, 1, 0, 1]), torch.zeros(4, dtype=torch.long)
    calls = {}
    for cls in CLASSES:
        for name, call in error_calls_class(getattr(R, cls), p4, t4, i4).items():
            calls[f"{cls}/{name}"] = call
    for fname in FUNCTIONALS:
        for name, call in error_calls_functional(getattr(F, fname), p4, t4).items():
            calls[f"{fname}/{name}"] = call
    return calls


def test_argument_errors_match_the_reference(ref):
    errors = ref["errors"]
    passed = []
    for name, call in _calls().items():
        if name in errors:
            kind, msg = errors[name]
            with pytest.raises(Exception) as info:
                call()
            assert type(info.value).__name__ == kind and str(info.value) == msg, (name, info.value)
        elif not name.startswith("retrieval_"):  # the functionals run kernels once their checks pass
            call()
            passed.append(name)
    # what the reference's loose checks let through is not rejected at construction here either
    for name in ("RetrievalAUROC/max_fpr_int_two", "RetrievalAUROC/max_fpr_neg", "RetrievalAUROC/top_k_zero"):
        assert name in passed or name in errors


def test_max_fpr_past_the_curve_raises_value_error_before_any_kernel():
    from metrics_b200.functional.retrieval import retrieval_auroc

    p, t = torch.tensor([.2, .7, .4]), torch.tensor([0, 1, 0])
    for bad in (2.0, 1.00000001, -0.5):
        with pytest.raises(ValueError, match="`max_fpr` must be 1 or lie in"):
            retrieval_auroc(p, t, max_fpr=bad)


def test_entry_points_reject_bad_arguments_before_any_launch():
    from metrics_b200 import _native

    lib = _native.lib()
    big = 1 << 20
    calls = {
        "top_k must be >= 0": lambda: lib.mb200_retrieval_auroc(8, 8, 8, 8, 4, -1, -1.0, 8, 8, 8, big, None),
        "max_fpr must be": lambda: lib.mb200_retrieval_auroc(8, 8, 8, 8, 4, 0, 1.5, 8, 8, 8, big, None),
        "NULL pointer": lambda: lib.mb200_retrieval_auroc(None, 8, 8, 8, 4, 0, -1.0, 8, 8, 8, big, None),
        "scratch too small": lambda: lib.mb200_retrieval_auroc(8, 8, 8, 8, 4, 0, 0.5, 8, 8, 8, 16, None),
        "bad size": lambda: lib.mb200_retrieval_auroc(8, 8, 8, 8, 0, 0, -1.0, 8, 8, 8, big, None),
        "max_k must be >= 1": lambda: lib.mb200_retrieval_pr_curve(8, 8, 8, 8, 4, 0, 0, 8, 8, 8, 8, big, None),
        "max_k must be >= 1, got -3": lambda: lib.mb200_retrieval_pr_curve(8, 8, 8, 8, 4, -3, 0, 8, 8, 8, 8, big, None),
        "NULL pointer ": lambda: lib.mb200_retrieval_pr_curve(8, 8, 8, 8, 4, 5, 0, 8, None, 8, 8, big, None),
        "scratch too small ": lambda: lib.mb200_retrieval_pr_curve(8, 8, 8, 8, 4, 5, 0, 8, 8, 8, 8, 40, None),
    }
    for msg, call in calls.items():
        before = lib.mb200_launch_count()
        assert call() == -1, msg
        assert lib.mb200_launch_count() == before, msg
        assert lib.mb200_last_error().decode().startswith(msg.strip()), (msg, lib.mb200_last_error())
    assert lib.mb200_retrieval_pr_curve_scratch_bytes(_native.RET_MAX_ELEMENTS + 1) == -1
    assert lib.mb200_retrieval_pr_curve_scratch_bytes(1000) > lib.mb200_retrieval_evaluate_scratch_bytes(1000)
