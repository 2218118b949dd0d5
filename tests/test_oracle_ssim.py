"""CPU: the two restatements of oracle/ssim.py — the numpy float64 oracle and the reference's torch op chain — against
the goldens made from the unmodified reference (tests/golden/ssim.npz)."""
import numpy as np
import pytest
import torch

from oracle import ssim as osm
from tests import ssim_cases as sc


def _per_image(case):
    """The functional's per-image values on the first batch, from the oracle: (sim, cs, map)."""
    kw = dict(case["kwargs"])
    p, t = case["batches"][0]
    args = {k: kw[k] for k in ("gaussian_kernel", "sigma", "kernel_size", "data_range") if k in kw}
    return osm.ssim(p, t, **args), args


SSIM_CASES = [c for c in sc.cases() if c["kind"] == "ssim"]
MS_CASES = [c for c in sc.cases() if c["kind"] == "ms"]


def _reduce(x, reduction):
    return {"elementwise_mean": np.mean, "sum": np.sum}.get(reduction, lambda v: v)(x)


@pytest.mark.parametrize("case", SSIM_CASES, ids=[c["name"] for c in SSIM_CASES])
def test_numpy_oracle_matches_the_goldens(case):
    golden = sc.load()
    (sim, cs, full), _ = _per_image(case)
    kw = case["kwargs"]
    red = kw.get("reduction", "elementwise_mean")
    assert np.allclose(_reduce(sim, red), golden[f"{case['name']}/functional"], atol=1e-12, rtol=0)
    if kw.get("return_contrast_sensitivity"):
        assert np.allclose(cs, golden[f"{case['name']}/functional_image"], atol=1e-12, rtol=0, equal_nan=True)
    if kw.get("return_full_image"):
        assert np.allclose(full, golden[f"{case['name']}/functional_image"], atol=1e-12, rtol=0)


@pytest.mark.parametrize("case", SSIM_CASES, ids=[c["name"] for c in SSIM_CASES])
def test_torch_chain_matches_the_goldens(case):
    golden = sc.load()
    _, args = _per_image(case)
    p, t = (torch.from_numpy(x) for x in case["batches"][0])
    sim, cs, full = osm.torch_chain_ssim(p, t, **args)
    kw = case["kwargs"]
    red = kw.get("reduction", "elementwise_mean")
    assert np.allclose(_reduce(sim.numpy(), red), golden[f"{case['name']}/functional"], atol=1e-12, rtol=0)
    if kw.get("return_contrast_sensitivity"):
        assert np.allclose(cs.numpy(), golden[f"{case['name']}/functional_image"], atol=1e-12, equal_nan=True)


@pytest.mark.parametrize("case", MS_CASES, ids=[c["name"] for c in MS_CASES])
def test_numpy_ms_oracle_matches_the_goldens(case):
    golden = sc.load()
    kw = dict(case["kwargs"])
    p, t = case["batches"][0]
    got = osm.ms_ssim(p, t, **{k: v for k, v in kw.items() if k != "reduction"})
    assert np.allclose(np.mean(got), golden[f"{case['name']}/functional"], atol=1e-12, rtol=0)


@pytest.mark.parametrize("level,noise", [(0.0, 1e-3), (100.0, 1e-3), (1000.0, 1e-2)])
def test_numpy_oracle_on_the_offset_workloads(level, noise):
    golden = sc.load()
    p, t = sc.offset_pair(level, noise)
    sim, _, _ = osm.ssim(p, t, data_range=1.0)
    # at level 1000 the reference's own float64 moments about zero lose about 1e-8; the oracle's are about the mean
    assert np.allclose(sim, golden[f"offset_{level:g}/f64"], atol=1e-7, rtol=0)


def test_unit_taps_reproduce_the_float64_reference_where_the_reference_taps_do_not():
    """At level 1000 the reference's float32 taps (total weight 1 − 1e-7) carried out exactly add about 0.06 to every
    variance; divided by their sum they give the float64 reference.  This is why K20 renormalises its taps."""
    golden = sc.load()
    p, t = sc.offset_pair(1000.0, 1e-2)
    taps = osm.filter_taps(osm.plan(4, True, 1.5, 11)[0], torch.float32)
    raw, _, _ = osm.ssim(p, t, data_range=1.0, taps=taps)
    unit, _, _ = osm.ssim(p, t, data_range=1.0, taps=taps, unit_taps=True)
    assert abs(unit - golden["offset_1000/f64"]).max() <= 1e-7
    assert abs(raw - golden["offset_1000/f64"]).max() > 0.1


def test_raw_taps_are_carried_exactly():
    """The default oracle with half-precision taps equals the reference's formula evaluated directly in float64."""
    rng = np.random.default_rng(0)
    p = rng.random((2, 1, 30, 34))
    t = p + 0.1 * rng.standard_normal(p.shape)
    taps = osm.filter_taps(osm.plan(4, True, 1.5, 11)[0], torch.bfloat16)
    sim, _, _ = osm.ssim(p, t, data_range=1.0, taps=taps)
    x, y = (np.pad(v, [(0, 0), (0, 0), (5, 5), (5, 5)], mode="reflect") for v in (p, t))

    def filt(img):
        for a, w in enumerate(taps):
            img = osm._correlate(img, w, a + 2)
        return img

    mx, my, mxx, myy, mxy = (filt(v) for v in (x, y, x * x, y * y, x * y))
    upper = 2 * (mxy - mx * my) + 9e-4
    lower = np.maximum(mxx - mx * mx, 0) + np.maximum(myy - my * my, 0) + 9e-4
    full = ((2 * mx * my + 1e-4) * upper) / ((mx * mx + my * my + 1e-4) * lower)
    assert np.abs(sim - full.reshape(2, -1).mean(1)).max() <= 1e-12
