"""GPU: kernel K21 (VIF-P and UQI on K20's moments) against the float64 numpy oracles (oracle/vif.py, oracle/uqi.py) on
the dtype-rounded inputs, and against the reference's op chains on the same GPU.

Tolerances (DESIGN.md K21): VIF per (image, channel) and its means 2e-5 relative for float32 and half-precision inputs
before the output rounding (plus one ulp of a half-precision output), 1e-10 for float64; UQI reduced values 1e-5
absolute (1e-10 float64), maps 1e-4 per pixel."""
import numpy as np
import pytest
import torch

from metrics_b200.functional.image import universal_image_quality_index as uqi
from metrics_b200.functional.image import visual_information_fidelity as vif
from metrics_b200.functional.image.vif import _vif_per_channel
from metrics_b200.image import UniversalImageQualityIndex, VisualInformationFidelity
from oracle import ssim as osm
from oracle import uqi as ouq
from oracle import vif as ovf

pytestmark = pytest.mark.gpu
DEV = "cuda"
HALF = (torch.float16, torch.bfloat16)


def _ulp(dtype):
    return {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}.get(dtype, 0.0)


def _pair(shape, dtype=torch.float32, seed=0, level=1.0, noise=0.1, flat=False):
    g = torch.Generator().manual_seed(seed)
    p = level * torch.rand(shape, generator=g, dtype=torch.float64)
    t = p + noise * level * torch.randn(shape, generator=g, dtype=torch.float64)
    if flat:  # a flat block (the σ < eps branches) and a block where target is minus preds (g < 0)
        h, w = shape[-2] // 2, shape[-1] // 2
        p[..., :h, :w], t[..., :h, :w] = 0.5 * level, 0.25 * level
        t[..., h:, w:] = level - p[..., h:, w:]
    return p.to(dtype), t.to(dtype)


def _vif_oracle(p, t, sigma_n_sq=2.0):
    dtype = p.dtype
    eps = torch.tensor(1e-10, dtype=dtype).item()
    sn = torch.tensor(sigma_n_sq, dtype=dtype).item()
    return ovf.vif_per_channel(p.cpu().double().numpy(), t.cpu().double().numpy(), sn, eps,
                               taps=ovf.filter_taps(dtype, DEV), round_to=dtype)


def _close(got, want, dtype, rel=2e-5, tol=None):
    got = got.double().cpu().numpy()
    tol = (tol if tol is not None else (1e-10 if dtype == torch.float64 else rel * np.abs(want))) + _ulp(dtype) * np.abs(want)
    both_nan = np.isnan(got) & np.isnan(want)
    assert np.all(both_nan | (np.abs(got - want) <= tol)), (got, want, np.abs(got - want).max())


VIF_CASES = [
    ("f32_41", (2, 3, 41, 41), torch.float32, 255.0, False),
    ("f64", (2, 3, 47, 63), torch.float64, 255.0, False),
    ("f16", (2, 2, 45, 47), torch.float16, 1.0, False),
    ("bf16", (2, 2, 45, 47), torch.bfloat16, 1.0, False),
    ("odd_c1", (3, 1, 53, 45), torch.float32, 255.0, False),
    ("flat_negative", (2, 2, 48, 50), torch.float32, 255.0, True),
    ("flat_negative_f64", (2, 2, 48, 50), torch.float64, 255.0, True),
    ("large", (1, 1, 517, 300), torch.float32, 255.0, False),
]


@pytest.mark.parametrize("name,shape,dtype,level,flat", VIF_CASES, ids=[c[0] for c in VIF_CASES])
def test_vif_matches_the_oracle(name, shape, dtype, level, flat):
    p, t = _pair(shape, dtype, level=level, flat=flat)
    want = _vif_oracle(p, t)
    pc, tc = p.to(DEV), t.to(DEV)
    got = _vif_per_channel(pc, tc, 2.0)
    assert got.dtype == dtype and got.shape == shape[:2]
    _close(got, want, dtype)
    _close(vif(pc, tc), np.asarray(want.mean()), dtype)


def test_vif_strided_views_and_sigma():
    p, t = _pair((4, 3, 50, 60), seed=4, level=255.0)
    pc, tc = p.to(DEV), t.to(DEV)
    for view in (lambda x: x[1:3], lambda x: x.contiguous(memory_format=torch.channels_last),
                 lambda x: x.transpose(2, 3)):
        _close(_vif_per_channel(view(pc), view(tc), 0.5), _vif_oracle(view(p), view(t), 0.5), torch.float32)


def test_vif_offset_images_keep_float32_accuracy():
    g = torch.Generator().manual_seed(3)
    ramp = torch.linspace(0, 1, 64, dtype=torch.float64)
    base = 1000.0 + ramp[:, None] + ramp[None, :]
    p = (base + 1e-2 * torch.randn(64, 64, generator=g, dtype=torch.float64))[None, None].float()
    t = (base + 1e-2 * torch.randn(64, 64, generator=g, dtype=torch.float64))[None, None].float()
    _close(_vif_per_channel(p.to(DEV), t.to(DEV), 2.0), _vif_oracle(p, t), torch.float32)
    _, crop = ouq.uqi(p.double().numpy(), t.double().numpy(), eps=float(torch.finfo(torch.float32).eps))
    assert abs(float(uqi(p.to(DEV), t.to(DEV))) - crop.mean()) <= 1e-5


UQI_CASES = [
    ("f32", (3, 3, 40, 52), torch.float32, {}),
    ("f64", (3, 3, 40, 52), torch.float64, {}),
    ("f16", (2, 3, 33, 47), torch.float16, {}),
    ("bf16", (2, 3, 33, 47), torch.bfloat16, {}),
    ("aniso", (2, 2, 45, 37), torch.float32, dict(kernel_size=(11, 5), sigma=(1.5, 0.8))),
    ("aniso2", (2, 2, 45, 37), torch.float64, dict(kernel_size=(3, 7), sigma=(0.7, 2.0))),
    ("one_tap", (2, 2, 30, 30), torch.float32, dict(kernel_size=(1, 1), sigma=(1.0, 1.0))),
    ("one_tap_axis", (2, 2, 30, 30), torch.float32, dict(kernel_size=(1, 5), sigma=(1.0, 1.0))),
    ("non_multiple", (2, 1, 97, 161), torch.float32, {}),
]


@pytest.mark.parametrize("name,shape,dtype,kw", UQI_CASES, ids=[c[0] for c in UQI_CASES])
def test_uqi_matches_the_oracle(name, shape, dtype, kw):
    p, t = _pair(shape, dtype, seed=5)
    ks, sg = kw.get("kernel_size", (11, 11)), kw.get("sigma", (1.5, 1.5))
    taps = osm.filter_taps(ouq.axes(ks, sg), dtype, DEV)
    full, crop = ouq.uqi(p.double().numpy(), t.double().numpy(), ks, sg, float(torch.finfo(dtype).eps), taps=taps,
                         unit_taps=True)
    pc, tc = p.to(DEV), t.to(DEV)
    tol = 1e-10 if dtype == torch.float64 else 1e-5
    got = uqi(pc, tc, reduction="none", **kw)
    assert got.shape == crop.shape and got.dtype == dtype
    _close(got, crop, dtype, tol=1e-4 if dtype != torch.float64 else 1e-10)
    _close(uqi(pc, tc, **kw), np.asarray(ouq.reduce(crop, "elementwise_mean")), dtype, tol=tol)
    _close(uqi(pc, tc, reduction="sum", **kw), np.asarray(crop.sum()), dtype, tol=tol * max(crop.size, 1))


def test_uqi_constant_target_and_flat_blocks():
    p, t = _pair((2, 2, 40, 40), seed=6, flat=True)
    t[1] = 0.5
    full, crop = ouq.uqi(p.double().numpy(), t.double().numpy(), taps=osm.filter_taps(ouq.axes(), torch.float32, DEV),
                         unit_taps=True)
    _close(uqi(p.to(DEV), t.to(DEV)), np.asarray(crop.mean()), torch.float32, tol=1e-5)


def test_agrees_with_the_op_chains_on_the_same_gpu():
    torch.backends.cudnn.allow_tf32 = False
    try:
        p, t = _pair((4, 3, 96, 80), seed=11)
        pc, tc = p.to(DEV), t.to(DEV)
        assert (_vif_per_channel(pc, tc, 2.0).double() - ovf.torch_chain_vif(pc, tc).double()).abs().max() <= 1e-4
        for ks, sg in (((11, 11), (1.5, 1.5)), ((3, 7), (0.7, 2.0))):
            chain = ouq.torch_chain_uqi(pc, tc, ks, sg)
            got = uqi(pc, tc, ks, sg, reduction="none")
            assert got.shape == chain.shape and (got - chain).abs().max() <= 1e-4
    finally:
        torch.backends.cudnn.allow_tf32 = True


def test_results_are_identical_from_run_to_run():
    p, t = _pair((4, 3, 130, 150), seed=9, level=255.0)
    pc, tc = p.to(DEV), t.to(DEV)
    assert torch.equal(_vif_per_channel(pc, tc, 2.0), _vif_per_channel(pc, tc, 2.0))
    assert torch.equal(uqi(pc, tc, reduction="sum"), uqi(pc, tc, reduction="sum"))
    assert torch.equal(uqi(pc, tc, reduction="none"), uqi(pc, tc, reduction="none"))


def test_an_update_does_not_synchronise_the_host():
    p, t = _pair((2, 3, 64, 64), seed=10)
    pc, tc = p.to(DEV), t.to(DEV)
    m1, m2 = VisualInformationFidelity().to(DEV), UniversalImageQualityIndex().to(DEV)
    m1.update(pc, tc)
    m2.update(pc, tc)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m1.update(pc, tc)
        m2.update(pc, tc)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_class_equals_functional_equals_summed_batches():
    batches = [_pair((2, c, 48, 52), seed=s) for s, c in ((0, 3), (1, 3))]
    gpu = [(p.to(DEV), t.to(DEV)) for p, t in batches]
    per = [_vif_per_channel(p, t, 2.0) for p, t in gpu]
    m = VisualInformationFidelity().to(DEV)
    for p, t in gpu:
        m.update(p, t)
    want = torch.cat([x.mean(1) for x in per]).sum() / 4
    assert abs(float(m.compute()) - float(want)) <= 1e-6
    assert torch.equal(vif(*gpu[0]), per[0].mean())
    for red in ("elementwise_mean", "sum"):
        m = UniversalImageQualityIndex(reduction=red).to(DEV)
        for p, t in gpu:
            m.update(p, t)
        total = sum(uqi(p, t, reduction="sum").double() for p, t in gpu)
        want = total if red == "sum" else total / (2 * 2 * 3 * 38 * 42)
        assert abs(float(m.compute()) - float(want)) <= 1e-5 * max(1.0, abs(float(want)))
    with pytest.warns(UserWarning):
        m = UniversalImageQualityIndex(reduction="none").to(DEV)
    for p, t in gpu:
        m.update(p, t)
    assert torch.equal(m.compute(), torch.cat([uqi(p, t, reduction="none") for p, t in gpu]))


def test_grad_mode_raises_in_functionals_and_forward_but_not_in_update():
    p, t = _pair((1, 1, 48, 48), seed=12)
    pc, tc = p.to(DEV).requires_grad_(True), t.to(DEV)
    for fn in (vif, uqi):
        with pytest.raises(RuntimeError, match="autograd graph"):
            fn(pc, tc)
    for cls in (VisualInformationFidelity, UniversalImageQualityIndex):
        with pytest.raises(RuntimeError, match="autograd graph"):
            cls().to(DEV)(pc, tc)
        cls().to(DEV).update(pc, tc)
    with torch.no_grad():
        vif(pc, tc)
        uqi(pc, tc)
