"""GPU: kernel K20 (structural similarity, MS-SSIM) against the float64 numpy oracle (oracle/ssim.py) on the
dtype-rounded inputs, and against the reference's op chain on the same GPU.

Tolerances per image (DESIGN.md K20): float32 and half-precision inputs 1e-5 absolute before the output rounding (plus
one ulp of a half-precision output), float64 1e-10, full maps 1e-4 per pixel."""
import numpy as np
import pytest
import torch

from metrics_b200.functional.image import (
    multiscale_structural_similarity_index_measure as msssim,
    structural_similarity_index_measure as ssim,
)
from metrics_b200.image import MultiScaleStructuralSimilarityIndexMeasure, StructuralSimilarityIndexMeasure
from oracle import ssim as osm

pytestmark = pytest.mark.gpu
DEV = "cuda"
HALF = (torch.float16, torch.bfloat16)


def _tol(dtype):
    return 1e-10 if dtype == torch.float64 else 1e-5


def _ulp(dtype):
    return {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}.get(dtype, 0.0)


def _pair(shape, dtype=torch.float32, seed=0, level=0.0, noise=0.1, tdtype=None):
    g = torch.Generator().manual_seed(seed)
    p = torch.rand(shape, generator=g, dtype=torch.float64) + level
    t = p + noise * torch.randn(shape, generator=g, dtype=torch.float64)
    return p.to(dtype), t.to(tdtype or dtype)


def _oracle(p, t, unit_taps=True, **kw):
    """Oracle on the inputs as K20 sees them: target rounded to preds' dtype, taps computed in preds' dtype on the GPU
    and, by default, divided by their sum as K20 divides them (DESIGN.md K20, deviation 3)."""
    axes, _ = osm.plan(p.ndim, kw.get("gaussian_kernel", True), kw.get("sigma", 1.5), kw.get("kernel_size", 11))
    taps = osm.filter_taps(axes, p.dtype, DEV)
    pn = p.cpu().double().numpy()
    tn = t.cpu().to(p.dtype).double().numpy()
    return osm.ssim(pn, tn, taps=taps, unit_taps=unit_taps, **kw)


def _close(got, want, dtype, tol=None):
    got = got.double().cpu().numpy()
    tol = (tol if tol is not None else _tol(dtype)) + _ulp(dtype) * np.abs(want)
    both_nan = np.isnan(got) & np.isnan(want)
    assert np.all(both_nan | (np.abs(got - want) <= tol)), (got, want, np.abs(got - want).max())


CASES = [
    ("f32", (3, 3, 40, 52), torch.float32, None, {}),
    ("f64", (3, 3, 40, 52), torch.float64, None, {}),
    ("f16", (3, 3, 40, 52), torch.float16, None, {}),
    ("bf16", (3, 3, 40, 52), torch.bfloat16, None, {}),
    ("mixed_target_f64", (2, 3, 33, 47), torch.float32, torch.float64, {}),
    ("mixed_target_f32_to_f16", (2, 3, 33, 47), torch.float16, torch.float32, {}),
    ("uniform", (2, 3, 40, 40), torch.float32, None, dict(gaussian_kernel=False, kernel_size=(5, 9))),
    ("anisotropic", (2, 2, 45, 37), torch.float32, None, dict(sigma=(0.8, 2.5))),
    ("one_tap_axis", (2, 2, 30, 30), torch.float32, None, dict(gaussian_kernel=False, kernel_size=(1, 7))),
    ("range_float", (2, 3, 40, 40), torch.float32, None, dict(data_range=1.0)),
    ("range_tuple_clamp", (2, 3, 40, 40), torch.float32, None, dict(data_range=(0.2, 0.7))),
    ("range_tuple_f16", (2, 3, 40, 40), torch.float16, None, dict(data_range=(0.2, 0.7))),
    ("smallest", (1, 1, 6, 6), torch.float32, None, {}),
    ("strip", (1, 1, 6, 8192), torch.float32, None, {}),
    ("non_multiple", (2, 1, 97, 161), torch.float32, None, {}),
    ("3d", (2, 2, 12, 20, 24), torch.float32, None, dict(kernel_size=(5, 5, 5), sigma=(1.0, 1.0, 1.0))),
    ("3d_gauss_ne_ks", (2, 1, 12, 20, 24), torch.float32, None, dict(kernel_size=(3, 3, 3), sigma=(0.8, 1.2, 1.5))),
    ("3d_uniform", (1, 2, 9, 10, 12), torch.float64, None, dict(gaussian_kernel=False, kernel_size=(3, 5, 3))),
]


@pytest.mark.parametrize("name,shape,dtype,tdtype,kw", CASES, ids=[c[0] for c in CASES])
def test_ssim_matches_the_oracle(name, shape, dtype, tdtype, kw):
    p, t = _pair(shape, dtype, tdtype=tdtype)
    want_s, want_cs, want_map = _oracle(p, t, **kw)
    pc, tc = p.to(DEV), t.to(DEV)
    got = ssim(pc, tc, reduction="none", **kw)
    assert got.dtype == dtype and got.shape == (shape[0],)
    _close(got, want_s, dtype)
    s2, cs = ssim(pc, tc, reduction="none", return_contrast_sensitivity=True, **kw)
    _close(cs, want_cs, dtype)
    s3, img = ssim(pc, tc, reduction="none", return_full_image=True, **kw)
    assert img.shape == want_map.shape and img.dtype == dtype
    _close(img, want_map, dtype, tol=1e-4)
    for red, fn in (("elementwise_mean", np.mean), ("sum", np.sum)):
        _close(ssim(pc, tc, reduction=red, **kw), np.asarray(fn(want_s)), dtype,
               tol=_tol(dtype) * shape[0] + _ulp(dtype) * abs(fn(want_s)) * 2)


@pytest.mark.parametrize("level,noise", [(0.0, 1e-3), (100.0, 1e-3), (1000.0, 1e-2)])
def test_offset_images_keep_float32_accuracy(level, noise):
    """A smooth ramp plus noise at a large level: E[x²] − E[x]² about zero loses everything in float32."""
    g = torch.Generator().manual_seed(3)
    ramp = torch.linspace(0, 1, 128, dtype=torch.float64)
    base = level + ramp[:, None] + ramp[None, :]
    p = (base + noise * torch.randn(128, 128, generator=g, dtype=torch.float64))[None, None].float()
    t = (base + noise * torch.randn(128, 128, generator=g, dtype=torch.float64))[None, None].float()
    want_s, want_cs, _ = _oracle(p, t, data_range=1.0)
    got, cs = ssim(p.to(DEV), t.to(DEV), data_range=1.0, reduction="none", return_contrast_sensitivity=True)
    _close(got, want_s, torch.float32)
    _close(cs, want_cs, torch.float32)


def test_large_batches_and_images():
    p, t = _pair((4096, 1, 16, 16), seed=1)
    want, _, _ = _oracle(p, t, data_range=1.0)
    _close(ssim(p.to(DEV), t.to(DEV), data_range=1.0, reduction="none"), want, torch.float32)
    p, t = _pair((1, 1, 4096, 4096), seed=2)
    got = ssim(p.to(DEV), t.to(DEV), reduction="none")
    want, _, _ = _oracle(p, t)
    _close(got, want, torch.float32)


def test_strided_views():
    p, t = _pair((4, 3, 37, 45), seed=4)
    want, _, _ = _oracle(p[1:3], t[1:3])
    pc, tc = p.to(DEV), t.to(DEV)
    _close(ssim(pc[1:3], tc[1:3], reduction="none"), want, torch.float32)  # batch slice
    cl_p = pc.contiguous(memory_format=torch.channels_last)
    cl_t = tc.contiguous(memory_format=torch.channels_last)
    want, _, _ = _oracle(p, t)
    _close(ssim(cl_p, cl_t, reduction="none"), want, torch.float32)
    pt, tt = p.transpose(2, 3), t.transpose(2, 3)
    want, _, _ = _oracle(pt, tt)
    _close(ssim(pc.transpose(2, 3), tc.transpose(2, 3), reduction="none"), want, torch.float32)


def test_nan_and_inf_pixels():
    p, t = _pair((3, 1, 30, 30), seed=5)
    p[0, 0, 3, 4] = float("nan")
    t[1, 0, 20, 20] = float("inf")
    want, _, want_map = _oracle(p, t, data_range=1.0)
    got, img = ssim(p.to(DEV), t.to(DEV), data_range=1.0, reduction="none", return_full_image=True)
    _close(got, want, torch.float32)
    assert torch.equal(torch.isnan(img.cpu()), torch.from_numpy(np.isnan(want_map)))
    # data_range=None: NaN in preds propagates to the range; NaN only in target is dropped by Python's max
    want_none, _, _ = _oracle(p, t)
    _close(ssim(p.to(DEV), t.to(DEV), reduction="none"), want_none, torch.float32)


@pytest.mark.parametrize("dtype", HALF)
def test_half_precision_stays_within_one_output_ulp_of_the_reference_taps(dtype):
    """Against the reference's own half-precision taps (total weight up to 1e-3 off 1, carried exactly by the oracle),
    renormalising them moves a per-image SSIM by less than one unit in the last place of the output dtype."""
    for kw in ({}, dict(data_range=1.0), dict(sigma=(0.8, 2.5))):
        p, t = _pair((3, 3, 40, 52), dtype, seed=13)
        want, _, _ = _oracle(p, t, unit_taps=False, **kw)
        _close(ssim(p.to(DEV), t.to(DEV), reduction="none", **kw), want, dtype)


def test_a_nan_at_the_tile_centre_keeps_the_other_windows_accurate_at_a_large_level():
    """The tile's shift falls back to a finite value of the tile: windows that do not touch the NaN keep float32
    accuracy at level 1000, where moments about zero would be off by more than 1."""
    g = torch.Generator().manual_seed(14)
    ramp = torch.linspace(0, 1, 96, dtype=torch.float64)
    base = 1000.0 + ramp[:, None] + ramp[None, :]
    p = (base + 1e-2 * torch.randn(96, 96, generator=g, dtype=torch.float64))[None, None].float()
    t = (base + 1e-2 * torch.randn(96, 96, generator=g, dtype=torch.float64))[None, None].float()
    p[0, 0, 16, 16] = float("nan")  # the centre of the first 32 x 32 tile
    t[0, 0, 48, 80] = float("inf")  # the centre of another tile, in the other input
    _, _, want = _oracle(p, t, data_range=1.0)
    _, img = ssim(p.to(DEV), t.to(DEV), data_range=1.0, return_full_image=True)
    got = img.double().cpu().numpy()
    assert np.array_equal(np.isfinite(got), np.isfinite(want))
    ok = np.isfinite(want)
    assert ok.sum() > 0.9 * ok.size
    # per image over the finite positions, as the per-image tolerance; moments about zero miss by 0.1 to 100 per pixel
    assert abs(got[ok].mean() - want[ok].mean()) <= 1e-5 and np.abs(got[ok] - want[ok]).max() <= 1e-2


def test_empty_batch_raises_as_the_reference():
    z = torch.zeros(0, 1, 16, 16, device=DEV)
    with pytest.raises(RuntimeError, match="numel"):
        ssim(z, z)
    with pytest.raises(IndexError, match="tuple index out of range"):
        ssim(z, z, data_range=1.0)


MS_CASES = [
    ("default", (2, 3, 180, 190), torch.float32, {}),
    ("range_none", (2, 1, 180, 180), torch.float32, dict(data_range=None)),
    ("betas3_simple", (2, 2, 64, 70), torch.float32, dict(betas=(0.2, 0.3, 0.5), normalize="simple", kernel_size=5,
                                                          sigma=0.8, data_range=1.0)),
    ("betas3_none", (2, 2, 64, 70), torch.float64, dict(betas=(0.2, 0.3, 0.5), normalize=None, kernel_size=5, sigma=0.8,
                                                        data_range=1.0)),
    ("minimum", (1, 1, 176, 176), torch.float32, dict(data_range=1.0)),
    ("3d", (1, 1, 16, 40, 40), torch.float32, dict(betas=(0.5, 0.5), kernel_size=3, sigma=0.5, data_range=1.0)),
    ("bf16", (2, 1, 180, 180), torch.bfloat16, dict(data_range=1.0)),
]


@pytest.mark.parametrize("name,shape,dtype,kw", MS_CASES, ids=[c[0] for c in MS_CASES])
def test_msssim_matches_the_oracle(name, shape, dtype, kw):
    p, t = _pair(shape, dtype, seed=7, noise=0.05)
    kw = {"data_range": 1.0, **kw}
    axes, _ = osm.plan(p.ndim, True, kw.get("sigma", 1.5), kw.get("kernel_size", 11))
    taps = osm.filter_taps(axes, dtype, DEV)
    okw = {k: v for k, v in kw.items()}
    want = osm.ms_ssim(p.double().numpy(), t.double().numpy(), taps=taps, round_to=dtype, unit_taps=True, **okw)
    got = msssim(p.to(DEV), t.to(DEV), reduction="none", **kw)
    assert got.dtype == torch.promote_types(dtype, torch.float32)
    _close(got, want, torch.float32 if dtype in HALF else dtype, tol=1e-5 if dtype != torch.float64 else 1e-10)


def test_classes_accumulate_over_updates():
    batches = [_pair((2, 3, 40, 40), seed=s) for s in range(3)]
    want = np.concatenate([_oracle(p, t, data_range=1.0)[0] for p, t in batches])
    for red in ("elementwise_mean", "sum", "none"):
        m = StructuralSimilarityIndexMeasure(data_range=1.0, reduction=red).to(DEV)
        for p, t in batches:
            m.update(p.to(DEV), t.to(DEV))
        ref = {"elementwise_mean": want.mean(), "sum": want.sum(), "none": want}[red]
        _close(m.compute(), np.asarray(ref), torch.float32, tol=1e-5 * 6)
    m = StructuralSimilarityIndexMeasure(data_range=1.0, return_contrast_sensitivity=True).to(DEV)
    for p, t in batches:
        m.update(p.to(DEV), t.to(DEV))
    sim, cs = m.compute()
    assert cs.shape == (6,)
    ms_batches = [_pair((1, 1, 180, 180), seed=s) for s in range(2)]
    ms_want = np.concatenate([osm.ms_ssim(p.numpy().astype(np.float64), t.numpy().astype(np.float64), data_range=1.0,
                                          taps=osm.filter_taps(osm.plan(4, True, 1.5, 11)[0], torch.float32, DEV),
                                          round_to=torch.float32, unit_taps=True) for p, t in ms_batches])
    m = MultiScaleStructuralSimilarityIndexMeasure(data_range=1.0).to(DEV)
    for p, t in ms_batches:
        m.update(p.to(DEV), t.to(DEV))
    _close(m.compute(), np.asarray(ms_want.mean()), torch.float32, tol=2e-5)


def test_results_are_identical_from_run_to_run():
    p, t = _pair((4, 3, 130, 150), seed=9)
    pc, tc = p.to(DEV), t.to(DEV)
    a = ssim(pc, tc, reduction="none", return_contrast_sensitivity=True)
    b = ssim(pc, tc, reduction="none", return_contrast_sensitivity=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert torch.equal(msssim(pc[..., :130, :130].repeat(1, 1, 2, 2), tc[..., :130, :130].repeat(1, 1, 2, 2)),
                       msssim(pc[..., :130, :130].repeat(1, 1, 2, 2), tc[..., :130, :130].repeat(1, 1, 2, 2)))


def test_an_update_does_not_synchronise_the_host():
    p, t = _pair((2, 3, 180, 180), seed=10)
    pc, tc = p.to(DEV), t.to(DEV)
    m1 = StructuralSimilarityIndexMeasure().to(DEV)
    m2 = MultiScaleStructuralSimilarityIndexMeasure().to(DEV)
    m1.update(pc, tc)  # warm-up: weights cached, module loaded
    m2.update(pc, tc)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m1.update(pc, tc)
        m2.update(pc, tc)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_agrees_with_the_op_chain_on_the_same_gpu():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for shape, kw in (((4, 3, 96, 80), {}), ((2, 2, 12, 20, 24), dict(kernel_size=(5, 5, 5), sigma=1.0)),
                          ((4, 3, 64, 64), dict(gaussian_kernel=False, kernel_size=7, data_range=(0.1, 0.9)))):
            p, t = _pair(shape, seed=11)
            pc, tc = p.to(DEV), t.to(DEV)
            cs_chain_s, cs_chain, _ = osm.torch_chain_ssim(pc, tc, **kw)
            got, cs = ssim(pc, tc, reduction="none", return_contrast_sensitivity=True, **kw)
            assert (got.double() - cs_chain_s.double()).abs().max() <= 1e-5
            assert (cs.double() - cs_chain.double()).abs().max() <= 1e-5
    finally:
        torch.backends.cudnn.allow_tf32 = True


def test_grad_mode_raises_in_functionals_and_forward_but_not_in_update():
    p, t = _pair((1, 1, 180, 180), seed=12)
    pc = p.to(DEV).requires_grad_(True)
    tc = t.to(DEV)
    with pytest.raises(RuntimeError, match="autograd graph"):
        ssim(pc, tc)
    with pytest.raises(RuntimeError, match="autograd graph"):
        msssim(pc, tc)
    for cls in (StructuralSimilarityIndexMeasure, MultiScaleStructuralSimilarityIndexMeasure):
        with pytest.raises(RuntimeError, match="autograd graph"):
            cls().to(DEV)(pc, tc)
        cls().to(DEV).update(pc, tc)  # update runs with grad disabled
    with torch.no_grad():
        ssim(pc, tc)
        msssim(pc, tc)
