"""CPU: the public surface of the structural-similarity classes and functionals against the reference's
(tests/golden/ssim_surface.json, dumped by tests/golden/make_golden_ssim.py), and the host layer — validation, error
precedence, states and reductions — replayed over every golden with the numpy oracle standing in for kernel K20."""
import importlib
import json
import os

import numpy as np
import pytest
import torch

from tests import ssim_cases as sc
from tests.conftest import GOLDEN_DIR
from tests.golden.make_golden_ssim import error_calls, ssim_states, ssim_surface


@pytest.fixture(scope="module")
def ref():
    return json.load(open(os.path.join(GOLDEN_DIR, "ssim_surface.json")))


@pytest.fixture
def host(monkeypatch):
    from metrics_b200 import _native

    monkeypatch.setattr(_native, "ssim", sc.standin_ssim)
    monkeypatch.setattr(_native, "ssim_avg_pool", sc.standin_pool)


def test_surface_matches_the_reference_but_for_is_differentiable(ref):
    ours = ssim_surface("metrics_b200")
    for name in ours:
        attrs = ours[name].get("attrs")
        if attrs is not None:
            assert attrs.pop("is_differentiable") == "False"
            assert ref["surface"][name]["attrs"].pop("is_differentiable") == "True"
    assert ours == ref["surface"]


def test_state_registry_matches_the_reference(ref):
    assert ssim_states("metrics_b200") == ref["states"]


def test_listed_in_both_packages():
    from metrics_b200 import image
    from metrics_b200.functional import image as fimage

    assert sorted(image.__all__) == ["MultiScaleStructuralSimilarityIndexMeasure", "StructuralSimilarityIndexMeasure"]
    assert sorted(fimage.__all__) == ["multiscale_structural_similarity_index_measure",
                                      "structural_similarity_index_measure"]


@pytest.mark.parametrize("case", sc.cases(), ids=[c["name"] for c in sc.cases()])
def test_goldens_through_classes_and_functionals_on_the_standin(host, case):
    F = importlib.import_module("metrics_b200.functional.image.ssim")  # noqa: N806
    S = importlib.import_module("metrics_b200.image.ssim")  # noqa: N806
    golden = sc.load()
    got = sc.run_case(case, F, S)
    assert set(got) == {k for k in golden if k.startswith(case["name"] + "/")}
    for key, value in got.items():
        want = golden[key]
        assert value.shape == want.shape and value.dtype == want.dtype, key
        assert np.allclose(value, want, rtol=0, atol=1e-10, equal_nan=True), (key, value, want)


def test_the_offset_goldens_show_the_reference_float32_collapse():
    golden = sc.load()
    for level, _ in ((0, 0), (100, 0), (1000, 0)):
        f64, f32 = golden[f"offset_{level:g}/f64"], golden[f"offset_{level:g}/f32"]
        assert (abs(f32 - f64).max() > 1) == (level > 0)


def test_error_types_messages_and_precedence(host, ref):
    F = importlib.import_module("metrics_b200.functional.image.ssim")  # noqa: N806
    S = importlib.import_module("metrics_b200.image.ssim")  # noqa: N806
    calls = error_calls(F, S)
    assert set(calls) == set(ref["errors"])
    for name, call in calls.items():
        kind, msg = ref["errors"][name]
        with pytest.raises(Exception) as info:
            call()
        assert type(info.value).__name__ == kind and str(info.value) == msg, (name, info.value)


def test_cpu_tensors_raise():
    from metrics_b200._native import NativeLibraryError
    from metrics_b200.functional.image import structural_similarity_index_measure

    x = torch.rand(1, 1, 16, 16)
    with pytest.raises(NativeLibraryError, match="CUDA tensors"):
        structural_similarity_index_measure(x, x)
