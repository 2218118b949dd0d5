"""CPU: the public surface of HausdorffDistance / hausdorff_distance against the reference's
(tests/golden/hausdorff_surface.json, dumped by tests/golden/make_golden_hausdorff.py), and the host layer — validation,
error precedence and the states — replayed over every golden with the numpy oracle standing in for kernel K19."""
import importlib
import json
import os

import pytest
import torch

from tests import hausdorff_cases as hc
from tests.conftest import GOLDEN_DIR
from tests.golden.make_golden_hausdorff import error_calls, hd_states, hd_surface


@pytest.fixture(scope="module")
def ref():
    return json.load(open(os.path.join(GOLDEN_DIR, "hausdorff_surface.json")))


@pytest.fixture
def host(monkeypatch):
    from metrics_b200 import _native

    monkeypatch.setattr(_native, "hausdorff_distance", hc.standin)


def test_surface_matches_the_reference(ref):
    assert hd_surface("metrics_b200") == ref["surface"]


def test_state_registry_matches_the_reference(ref):
    assert hd_states("metrics_b200") == ref["states"]


def test_importable_from_both_packages_but_not_listed():
    from metrics_b200 import segmentation
    from metrics_b200.functional import segmentation as fseg
    from metrics_b200.functional.segmentation import hausdorff_distance  # noqa: F401
    from metrics_b200.segmentation import HausdorffDistance  # noqa: F401

    assert "HausdorffDistance" not in segmentation.__all__ and "hausdorff_distance" not in fseg.__all__


def test_goldens_through_classes_and_functionals_on_the_standin(host):
    golden = hc.load()
    for case in hc.cases():
        hc.check_case(golden, case, "cpu")


def test_error_types_messages_and_precedence(host, ref):
    F = importlib.import_module("metrics_b200.functional.segmentation.hausdorff_distance")  # noqa: N806
    S = importlib.import_module("metrics_b200.segmentation.hausdorff_distance")  # noqa: N806
    calls = error_calls(F, S)
    assert set(calls) == set(ref["errors"])
    for name, call in calls.items():
        kind, msg = ref["errors"][name]
        with pytest.raises(Exception) as info:
            call()
        assert type(info.value).__name__ == kind and str(info.value) == msg, (name, info.value)


def test_a_raising_update_leaves_the_states_unchanged(host):
    from metrics_b200.segmentation import HausdorffDistance

    ok = torch.ones(2, 3, 6, 6, dtype=torch.int64)
    ok[:, :, 2:4, 2:4] = 0
    empty, bad = ok.clone(), ok.clone()
    empty[1, 2] = 0
    bad[0, 1, 0, 0] = 5
    lab = torch.randint(0, 3, (2, 6, 6))
    for m, good, fails in ((HausdorffDistance(3), (ok, ok), [(empty, empty), (bad, ok), (ok, bad)]),
                           (HausdorffDistance(3, input_format="index"), (lab, lab), [(lab, lab + 3), (lab - 1, lab)])):
        m.update(*good)
        before = {k: v.clone() for k, v in m.metric_state.items()}
        for p, t in fails:
            with pytest.raises((RuntimeError, ValueError)):
                m.update(p, t)
            assert all(torch.equal(before[k], v) for k, v in m.metric_state.items())


def test_empty_batch_and_empty_images(host):
    from metrics_b200.functional.segmentation import hausdorff_distance

    assert hausdorff_distance(torch.zeros(0, 3, 4, 4, dtype=torch.bool), torch.zeros(0, 3, 4, 4, dtype=torch.bool),
                              3).shape == (0, 2)
    with pytest.raises(RuntimeError, match="numel"):
        hausdorff_distance(torch.zeros(1, 3, 0, 4, dtype=torch.bool), torch.zeros(1, 3, 0, 4, dtype=torch.bool), 3)


def test_cpu_tensors_raise():
    from metrics_b200._native import NativeLibraryError
    from metrics_b200.functional.segmentation import hausdorff_distance

    x = torch.ones(1, 2, 4, 4, dtype=torch.bool)
    with pytest.raises(NativeLibraryError, match="CUDA tensors"):
        hausdorff_distance(x, x, 2)
