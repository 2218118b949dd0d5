"""CPU: VIF and UQI (kernel K21).  The float64 oracles (oracle/vif.py, oracle/uqi.py) and the reference's torch chains
against the goldens made from the unmodified reference (tests/golden/vif_uqi.npz); the public surface, state registries
and error paths against tests/golden/vif_uqi_surface.json; every golden replayed through the classes and functionals
with the oracles standing in for the kernels; and the C-ABI of the three new entry points."""
import ctypes
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
from tests.test_abi import _patch_host

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


# ---- C-ABI ------------------------------------------------------------------------------------------------------------
STREAM = 0xCAFE
NEW = ("mb200_vif_scale_update", "mb200_vif_decimate", "mb200_uqi_update")


class _Recorder:
    def __init__(self):
        self.calls = {}
        for name, (ret, args) in _native.IMAGE_SIGNATURES.items():
            def callback(*values, _name=name):
                self.calls.setdefault(_name, []).append(values)
                return 4096 if _name.endswith("_bytes") else 0

            setattr(self, name, ctypes.CFUNCTYPE(_native._C_TYPES[ret], *[_native._C_TYPES[a] for a in args])(callback))


def _drives():
    p = torch.zeros(2, 3, 41, 45).contiguous(memory_format=torch.channels_last)
    t = torch.zeros(2, 3, 45, 41).transpose(2, 3)
    w = torch.ones(40)
    return p, t, w, (
        lambda: _native.vif_scale(p, t, w, (1, 17, 17), 1e-10, 2.0),
        lambda: _native.vif_decimate(p, t, w, (9, 9)),
        lambda: _native.uqi(p, t, w, (1, 11, 5), (0, 2, 5), (5, 2), 1e-7, True),
    )


def test_new_wrappers_call_the_abi_as_declared(monkeypatch):
    fake = _Recorder()
    monkeypatch.setattr(_native, "lib", lambda: fake)
    _patch_host(monkeypatch, STREAM)
    p, t, w, (scale, decimate, uqi) = _drives()
    a, b = scale()
    assert a.shape == b.shape == (2, 3) and a.dtype == torch.float64
    po, to = decimate()
    assert po.shape == to.shape == (2, 3, 17, 19) and po.dtype == torch.float32  # ceil((41 - 9 + 1) / 2), (45 - 9 + 2) // 2
    sums, img = uqi()
    assert sums.shape == (2,) and img.shape == (2, 3, 1, 41 + 4 - 11 + 1, 45 + 10 - 5 + 1)
    for name in NEW:
        (call,) = fake.calls[name]
        assert len(call) == len(_native.IMAGE_SIGNATURES[name][1]) and call[-1] == STREAM
        assert call[1] == _native.F32 and call[3] == _native.F32 and call[4:9] == (2, 3, 1, 41, 45)
        assert call[9:14] == (p.stride(0), p.stride(1), 0, p.stride(2), p.stride(3))
        assert call[14:19] == (t.stride(0), t.stride(1), 0, t.stride(2), t.stride(3))
    vs, dc, uq = (fake.calls[n][0] for n in NEW)
    assert vs[19:22] == (1, 17, 17) and vs[23:25] == (1e-10, 2.0) and vs[-2] == 4096
    assert dc[19:21] == (9, 9) and all(v is not None for v in dc[21:24])
    assert uq[19:27] == (1, 11, 5, 0, 2, 5, 5, 2) and uq[28] == 1e-7 and uq[30] is not None and uq[-2] == 4096


def test_real_library_accepts_the_new_wrappers_arguments_up_to_the_first_cuda_call(monkeypatch):
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present: host pointers must not reach the kernels")
    _patch_host(monkeypatch, 0)
    for drive in _drives()[3]:
        with pytest.raises(_native.NativeLibraryError, match=r"\(code -2\): CUDA error"):
            drive()


@pytest.mark.parametrize("bad", [-1, _native.I64, _native.I32, _native.U8, _native.BOOL, 10])
def test_new_entry_points_reject_non_float_dtype_tags_before_any_launch(bad):
    lib = _native.lib()
    geo = (1, 1, 1, 48, 48) + (2304, 2304, 0, 48, 1) * 2
    for which, msg in ((0, f"preds must be a floating-point tensor (dtype tag {bad})"),
                       (1, f"target must be a floating-point tensor (dtype tag {bad})")):
        tags = (bad, _native.F32) if which == 0 else (_native.F32, bad)
        for rc in (lib.mb200_vif_scale_update(8, tags[0], 8, tags[1], *geo, 1, 17, 17, 8, 1e-10, 2.0, 8, 8, 16, 1 << 20,
                                              None),
                   lib.mb200_vif_decimate(8, tags[0], 8, tags[1], *geo, 9, 9, 8, 8, 8, None),
                   lib.mb200_uqi_update(8, tags[0], 8, tags[1], *geo, 1, 11, 11, 0, 5, 5, 5, 5, 8, 1e-7, 8, None, 16,
                                        1 << 20, None)):
            assert rc == -1 and lib.mb200_last_error().decode() == msg


def test_new_entry_points_reject_bad_geometry_before_any_launch():
    lib = _native.lib()
    geo = (1, 1, 1, 48, 48) + (2304, 2304, 0, 48, 1) * 2
    small = (1, 1, 1, 16, 16) + (256, 256, 0, 16, 1) * 2
    f = _native.F32
    checks = [
        (lambda: lib.mb200_vif_scale_update(8, f, 8, f, *geo, 1, 0, 17, 8, 1e-10, 2.0, 8, 8, 16, 1 << 20, None), "tap counts"),
        (lambda: lib.mb200_vif_scale_update(8, f, 8, f, *geo, 1, 256, 17, 8, 1e-10, 2.0, 8, 8, 16, 1 << 20, None), "tap counts"),
        (lambda: lib.mb200_vif_scale_update(8, f, 8, f, *small, 1, 17, 17, 8, 1e-10, 2.0, 8, 8, 16, 1 << 20, None), "empty output"),
        (lambda: lib.mb200_vif_decimate(8, f, 8, f, *small, 17, 9, 8, 8, 8, None), "empty output"),
        (lambda: lib.mb200_vif_decimate(8, f, 8, f, *geo, 0, 9, 8, 8, 8, None), "tap counts"),
        (lambda: lib.mb200_uqi_update(8, f, 8, f, *small, 1, 11, 11, 0, 16, 5, 5, 5, 8, 1e-7, 8, None, 16, 1 << 20, None),
         "reflect pads"),
        (lambda: lib.mb200_uqi_update(8, f, 8, f, *small, 1, 11, 11, 0, 5, 5, -1, 5, 8, 1e-7, 8, None, 16, 1 << 20, None),
         "crop margins"),
        (lambda: lib.mb200_uqi_update(8, f, 8, f, *small, 1, 41, 11, 0, 5, 5, 5, 5, 8, 1e-7, 8, None, 16, 1 << 20, None),
         "empty output"),
    ]
    for call, msg in checks:
        assert call() == -1 and msg in lib.mb200_last_error().decode(), msg
