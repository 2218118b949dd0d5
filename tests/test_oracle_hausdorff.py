"""CPU: the numpy oracle of kernel K19 against the reference's goldens (bit for bit) and, on non-square images where the
reference is wrong, against scipy.ndimage distance transforms evaluated at the edge pixels."""
import numpy as np
import pytest
import torch
from scipy import ndimage

from oracle import hausdorff as oh
from tests import hausdorff_cases as hc

CASES = hc.cases()


@pytest.fixture(scope="module")
def golden():
    return hc.load()


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_oracle_matches_the_reference_goldens(golden, case):
    kw = dict(case["kwargs"])
    fmt = kw.pop("input_format", "one-hot")
    (p, t), _ = hc.tensors(case)
    got = oh.hausdorff(p.numpy(), t.numpy(), kw.pop("num_classes"), kw.get("include_background", False),
                       kw.get("distance_metric", "euclidean"), kw.get("spacing"), kw.get("directed", False), fmt)
    want = golden[f"{case['name']}/functional"]
    assert got.dtype == np.float32 and hc.ulps(got, want) <= hc.golden_ulps(case), (got, want)


def test_reference_sqrt_is_the_only_difference(golden):
    """Where a euclidean golden differs from the oracle, the oracle is the correctly rounded square root of the
    reference's own float32 sum of squares (recomputed in float64 from the same terms)."""
    differ = 0
    for case in CASES:
        if hc.golden_ulps(case) == 0:
            continue
        kw = dict(case["kwargs"])
        (p, t), _ = hc.tensors(case)
        got = oh.hausdorff(p.numpy(), t.numpy(), kw["num_classes"], kw.get("include_background", False), "euclidean",
                           kw.get("spacing"), kw.get("directed", False), kw.get("input_format", "one-hot"))
        want = golden[f"{case['name']}/functional"]
        for g, w in zip(got.ravel(), want.ravel()):
            if g != w:
                differ += 1
                square = np.float64(g) ** 2  # an exact float32 sum of squares lies within half an ulp of g's square
                assert abs(np.sqrt(square) - g) <= abs(np.sqrt(square) - w)
    assert differ < 20


def _scipy(p, t, metric, sampling):
    ep, et = oh.edges(p), oh.edges(t)
    if metric == "euclidean":
        dt = [ndimage.distance_transform_edt(~e, sampling=sampling) for e in (et, ep)]
    else:
        dt = [ndimage.distance_transform_cdt(~e, metric=metric) for e in (et, ep)]
    return max(dt[0][ep].max(), dt[1][et].max())


@pytest.mark.parametrize("shape", [(7, 19), (19, 7), (3, 40), (40, 3), (12, 13)])
@pytest.mark.parametrize("metric,sampling", [("euclidean", (1, 1)), ("euclidean", (0.7, 1.3)), ("chessboard", (1, 1)),
                                             ("taxicab", (1, 1))])
def test_oracle_matches_scipy_on_non_square_images(shape, metric, sampling):
    rng = np.random.default_rng(sum(shape))
    for _ in range(20):
        p, t = rng.random(shape) < 0.3, rng.random(shape) < 0.3
        if not p.any() or not t.any():
            continue
        spacing = [v if v != 1 else 1 for v in sampling]
        got = oh.pair_distance(p, t, spacing, metric, False)
        assert np.isclose(got, _scipy(p, t, metric, sampling), rtol=1e-6, atol=0), (p, t)


def test_column_nearest_mode_equals_the_brute_force(monkeypatch):
    rng = np.random.default_rng(5)
    for metric in hc.METRICS:
        for spacing in ([1, 1], [2, 3], [0.7, 1.3], [1, 0.37]):
            p, t = rng.random((30, 41)) < 0.2, rng.random((30, 41)) < 0.05
            want = oh.pair_distance(p, t, spacing, metric, False)
            monkeypatch.setattr(oh, "BRUTE_LIMIT", 0)
            got = oh.pair_distance(p, t, spacing, metric, False)
            monkeypatch.undo()
            assert got.view(np.uint32) == want.view(np.uint32), (metric, spacing)


def test_edges_and_empty_sides():
    m = np.zeros((5, 5), bool)
    m[1:4, 1:4] = True
    e = oh.edges(m)
    assert e.sum() == 8 and not e[2, 2]
    assert oh.edges(np.ones((1, 1), bool)).all()
    assert oh.pair_distance(m, np.zeros_like(m), [1, 1], "euclidean", True) == np.inf
    assert oh.pair_distance(np.zeros_like(m), np.zeros_like(m), [1, 1], "euclidean", False) is None


def test_torch_chain_matches_the_oracle_on_non_square_images():
    rng = np.random.default_rng(3)
    for shape in ((9, 17), (17, 9)):
        for metric in hc.METRICS:
            p, t = rng.random(shape) < 0.3, rng.random(shape) < 0.3
            got = oh.chain_pair(torch.from_numpy(p), torch.from_numpy(t), [0.7, 1.3], metric, False)
            want = oh.pair_distance(p, t, [0.7, 1.3], metric, False)
            assert got.item() == float(want)
