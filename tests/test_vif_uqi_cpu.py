"""CPU: VIF and UQI (kernel K21).  The float64 oracles (oracle/vif.py, oracle/uqi.py) and the reference's torch chains
against the goldens made from the unmodified reference (tests/golden/vif_uqi.npz); the public surface, state registries
and error paths against tests/golden/vif_uqi_surface.json; every golden replayed through the classes and functionals
with the oracles standing in for the kernels.  The C-ABI of K21 is checked in tests/test_abi.py,
tests/test_dtype_dispatch_abi.py and tests/test_image_abi.py."""
import json
import os
import warnings

import numpy as np
import pytest
import torch

from metrics_b200 import _native
from oracle import uqi as ouq
from oracle import vif as ovf
from tests import vif_uqi_cases as vc
from tests.conftest import GOLDEN_DIR
from tests.golden.make_golden_vif_uqi import error_calls, modules, states, surface

CASES = vc.cases()
IDS = [c["name"] for c in CASES]
F64 = [c for c in CASES if c["dtype"] == "f64"]


@pytest.fixture(scope="module")
def ref():
    return json.load(open(os.path.join(GOLDEN_DIR, "vif_uqi_surface.json")))


@pytest.fixture
def host(monkeypatch):
    monkeypatch.setattr(_native, "vif_scale", vc.standin_vif_scale)
    monkeypatch.setattr(_native, "vif_decimate", vc.standin_vif_decimate)
    monkeypatch.setattr(_native, "uqi", vc.standin_uqi)


def _oracle_functional(case):
    p, t = case["batches"][0]
    kw = case["kwargs"]
    if case["kind"] == "vif":
        return np.mean(ovf.vif_per_channel(p, t, kw.get("sigma_n_sq", 2.0)))
    _, crop = ouq.uqi(p, t, kw.get("kernel_size", (11, 11)), kw.get("sigma", (1.5, 1.5)), eps=float(np.finfo(np.float64).eps))
    return ouq.reduce(crop, kw.get("reduction", "elementwise_mean"))


def _tol(case):
    return 1e-2 if case["name"] == "uqi_flat_negative" else 1e-10


@pytest.mark.parametrize("case", F64, ids=[c["name"] for c in F64])
def test_numpy_oracle_matches_the_goldens(case):
    """Exact but for UQI's flat blocks: there the reference's float64 variances are cancellation noise of about 1e-17,
    the size of float64's eps in UQI's denominator, so they move its map; the oracle's are 0."""
    got, want = _oracle_functional(case), vc.load()[f"{case['name']}/functional"]
    assert np.shape(got) == want.shape
    assert np.allclose(got, want, rtol=0, atol=_tol(case), equal_nan=True)


@pytest.mark.parametrize("case", F64, ids=[c["name"] for c in F64])
def test_torch_chains_match_the_goldens(case):
    p, t = (torch.from_numpy(x) for x in case["batches"][0])
    kw = case["kwargs"]
    want = vc.load()[f"{case['name']}/functional"]
    if case["kind"] == "vif":
        got = ovf.torch_chain_vif(p, t, kw.get("sigma_n_sq", 2.0)).mean().numpy()
    else:
        got = ouq.reduce(ouq.torch_chain_uqi(p, t, kw.get("kernel_size", (11, 11)), kw.get("sigma", (1.5, 1.5))).numpy(),
                         kw.get("reduction", "elementwise_mean"))
    assert np.allclose(got, want, rtol=0, atol=1e-12, equal_nan=True)


def test_the_offset_goldens_show_the_reference_float32_collapse():
    """At level 1000 the reference's float32 VIF and UQI are far from its float64 values; the oracle is not."""
    golden = vc.load()
    for level in (0, 100, 1000):
        p, t = vc.offset_pair(float(level), 1e-2)
        assert abs(np.mean(ovf.vif_per_channel(p, t)) - golden[f"offset_{level}/vif_f64"]) <= 1e-7
        _, crop = ouq.uqi(p, t, eps=float(np.finfo(np.float64).eps))
        assert abs(np.mean(crop) - golden[f"offset_{level}/uqi_f64"]) <= 1e-7
    for kind in ("vif", "uqi"):
        assert abs(golden[f"offset_0/{kind}_f32"] - golden[f"offset_0/{kind}_f64"]) < 1e-3
        assert abs(golden[f"offset_1000/{kind}_f32"] - golden[f"offset_1000/{kind}_f64"]) > 0.1


def test_surface_matches_the_reference_but_for_is_differentiable(ref):
    ours = surface("metrics_b200")
    for name in ours:
        attrs = ours[name].get("attrs")
        if attrs is not None:
            assert attrs.pop("is_differentiable") == "False"
            assert ref["surface"][name]["attrs"].pop("is_differentiable") == "True"
    assert ours == ref["surface"]


def test_state_registry_matches_the_reference(ref):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        assert states("metrics_b200") == ref["states"]


def test_importable_from_both_packages_but_not_listed():
    from metrics_b200 import image
    from metrics_b200.functional import image as fimage

    assert image.VisualInformationFidelity and image.UniversalImageQualityIndex
    assert fimage.visual_information_fidelity and fimage.universal_image_quality_index
    assert "VisualInformationFidelity" not in image.__all__ and "visual_information_fidelity" not in fimage.__all__


def test_error_types_messages_and_precedence(host, ref):
    calls = error_calls(modules("metrics_b200"))
    assert set(calls) == set(ref["errors"])
    for name, call in calls.items():
        kind, msg = ref["errors"][name]
        with pytest.raises(Exception) as info:
            call()
        assert type(info.value).__name__ == kind and str(info.value) == msg, (name, info.value)


def test_none_reduction_warns_as_the_reference():
    from metrics_b200.image import UniversalImageQualityIndex

    with pytest.warns(UserWarning, match="will save all targets and predictions"):
        UniversalImageQualityIndex(reduction="none")


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_goldens_through_classes_and_functionals_on_the_standin(host, case):
    golden = vc.load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = vc.run_case(case, *modules("metrics_b200")["vif"], *modules("metrics_b200")["uqi"])
    assert set(got) == {k for k in golden if k.startswith(case["name"] + "/")}
    for key, value in got.items():
        want = golden[key]
        assert value.shape == want.shape and value.dtype == want.dtype, key
        if case["dtype"] == "f64":
            assert np.allclose(value, want, rtol=0, atol=_tol(case), equal_nan=True), (key, value, want)

