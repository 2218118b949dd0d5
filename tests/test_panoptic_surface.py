"""CPU: the public surface of the panoptic qualities against the reference's (tests/golden/panoptic_surface.json, dumped by
tests/golden/make_golden_panoptic.py) — functional signatures, the state registry of both classes, and the host
validation's exceptions and messages.  tests/test_api_surface.py covers the class surface."""
import json
import os

import pytest
import torch

from tests import panoptic_cases as pc
from tests.conftest import GOLDEN_DIR
from tests.golden.make_golden_panoptic import pq_states, pq_surface


@pytest.fixture(scope="module")
def ref():
    return json.load(open(os.path.join(GOLDEN_DIR, "panoptic_surface.json")))


def test_functional_surface_matches_the_reference(ref):
    assert pq_surface("metrics_b200") == ref["surface"]


def test_functional_detection_exports_only_the_panoptic_qualities():
    from metrics_b200.functional import detection

    assert sorted(detection.__all__) == ["modified_panoptic_quality", "panoptic_quality"]


def test_state_registry_matches_the_reference(ref):
    assert pq_states("metrics_b200") == ref["states"]


def test_validation_errors_match_the_reference(ref):
    from metrics_b200.detection import PanopticQuality
    from metrics_b200.functional.detection import panoptic_quality

    p0, t0 = pc.inputs0()
    calls = {
        "things_not_int": lambda: panoptic_quality(p0, t0, {0, 1.0}, {6, 7}),
        "stuffs_not_int": lambda: panoptic_quality(p0, t0, {0, 1}, {6, "7"}),
        "overlap": lambda: panoptic_quality(p0, t0, {0, 1}, {1, 7}),
        "empty": lambda: PanopticQuality(set(), set()),
        "preds_type": lambda: panoptic_quality(p0.numpy(), t0, {0, 1}, {6, 7}),
        "target_type": lambda: panoptic_quality(p0, [1], {0, 1}, {6, 7}),
        "shape": lambda: panoptic_quality(p0, t0[:, :3], {0, 1}, {6, 7}),
        "dims": lambda: panoptic_quality(p0[0, 0], t0[0, 0], {0, 1}, {6, 7}),
        "last_dim": lambda: panoptic_quality(p0[..., :1], t0[..., :1], {0, 1}, {6, 7}),
    }
    assert set(calls) | {"unknown_preds"} == set(ref["errors"])
    for name, call in calls.items():
        kind, msg = ref["errors"][name]
        with pytest.raises(Exception) as info:
            call()
        assert type(info.value).__name__ == kind and str(info.value) == msg, (name, info.value)


def test_duplicate_categories_warn():
    from metrics_b200.detection import ModifiedPanopticQuality

    with pytest.warns(UserWarning, match="`things` categories contained duplicates"):
        m = ModifiedPanopticQuality([1, 1, 2], [5])
    assert m.things == {1, 2} and m.void_color == (6, 0) and m.cat_id_to_continuous_id == {1: 0, 2: 1, 5: 2}


@pytest.mark.parametrize("dtype", [torch.float32, torch.bool])
def test_floating_and_bool_inputs_raise(dtype):
    from metrics_b200.functional.detection import panoptic_quality

    x = torch.zeros(1, 3, 3, 2, dtype=dtype)
    with pytest.raises(ValueError, match="integer"):
        panoptic_quality(x, x, {0}, {1})


def test_cpu_tensors_raise():
    from metrics_b200._native import NativeLibraryError
    from metrics_b200.functional.detection import modified_panoptic_quality

    p, t = pc.inputs0()
    with pytest.raises(NativeLibraryError, match="CUDA tensors"):
        modified_panoptic_quality(p, t, {0, 1}, {6, 7})
