"""GPU: kernel K19 (Hausdorff distance) — the [N, C'] distances equal to the numpy oracle with torch.equal (inf included)
over every input format, dtype, layout, metric, spacing and directedness, image sizes around every launch boundary,
non-square images, tall images, float32 rounding of large distances, the pruning worst case and the scratch chunking;
equal to the reference's op chain on the same GPU; the goldens through the class and the functional; the errors and
run-to-run bits."""
import numpy as np
import pytest
import torch

from metrics_b200 import _native
from oracle import hausdorff as oh
from tests import hausdorff_cases as hc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = hc.cases()


def _run(p, t, num_classes, **kw):
    from metrics_b200.functional.segmentation import hausdorff_distance

    got = hausdorff_distance(p.to(DEV), t.to(DEV), num_classes, **kw)
    assert got.dtype == torch.float32 and got.device.type == "cuda"
    return got.cpu()


def _want(p, t, num_classes, **kw):
    return torch.from_numpy(oh.hausdorff(p.numpy(), t.numpy(), num_classes, kw.get("include_background", False),
                                         kw.get("distance_metric", "euclidean"), kw.get("spacing"),
                                         kw.get("directed", False), kw.get("input_format", "one-hot")))


def _check(p, t, num_classes, **kw):
    got, want = _run(p, t, num_classes, **kw), _want(p, t, num_classes, **kw)
    assert torch.equal(got, want), (got, want, (got - want).abs().max())


def _masks(shape, seed, density=0.25):
    rng = np.random.default_rng(seed)
    n, c, h, w = shape
    side = max(h, w)
    m = hc.blobs(rng, n, c, side, density)[:, :, :h, :w].copy()
    m[..., 0, 0] = True  # never empty after the crop
    return torch.from_numpy(m)


@pytest.fixture(scope="module")
def golden():
    return hc.load()


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_goldens_through_the_class_and_the_functional(golden, case):
    hc.check_case(golden, case, DEV)


@pytest.mark.parametrize("shape", [(3, 4, 37, 53), (3, 4, 53, 37)])
@pytest.mark.parametrize("spacing", hc.SPACINGS, ids=["none", "int", "float", "mixed"])
@pytest.mark.parametrize("metric", hc.METRICS)
@pytest.mark.parametrize("directed", [False, True])
def test_metrics_spacings_and_non_square_images(shape, spacing, metric, directed):
    p, t = _masks(shape, 1).long(), _masks(shape, 2).long()
    _check(p, t, 4, distance_metric=metric, spacing=spacing, directed=directed)


@pytest.mark.parametrize("dtypes", [(d, d) for d in hc.ONE_HOT_DTYPES] + [(torch.uint8, torch.int32), (torch.bool, torch.int8)],
                         ids=lambda d: f"{d[0]}-{d[1]}".replace("torch.", ""))
@pytest.mark.parametrize("layout", ["planar", "channels_last", "strided"])
def test_one_hot_dtypes_and_layouts(dtypes, layout):
    p, t = _masks((3, 3, 29, 41), 3).to(dtypes[0]), _masks((3, 3, 29, 41), 4).to(dtypes[1])
    want = _want(p.long(), t.long(), 3, include_background=True, spacing=[0.7, 1.3])
    if layout == "channels_last":
        p, t = p.to(memory_format=torch.channels_last), t.to(memory_format=torch.channels_last)
    elif layout == "strided":
        p, t = torch.cat([p, p], 3)[..., ::2], torch.cat([t, t], 2).transpose(2, 3).contiguous().transpose(2, 3)[:, :, :29]
        want = _want(p.long(), t.long(), 3, include_background=True, spacing=[0.7, 1.3])
    got = _run(p, t, 3, include_background=True, spacing=[0.7, 1.3])
    assert torch.equal(got, want)


@pytest.mark.parametrize("include_background", [False, True])
@pytest.mark.parametrize("transposed", [False, True])
def test_index_format(include_background, transposed):
    g = torch.Generator().manual_seed(7)
    lab = torch.randint(0, 5, (4, 33, 47), generator=g)
    lab2 = torch.roll(lab, (1, 3), (1, 2))
    lab2[0, :5] = 0  # some classes absent from one side somewhere: inf
    if transposed:
        lab, lab2 = lab.transpose(1, 2), lab2.transpose(1, 2)
    for c in range(5):  # every class present on at least one side of every sample
        lab[:, 0, c] = c
    _check(lab, lab2, 5, include_background=include_background, input_format="index", distance_metric="chessboard")


@pytest.mark.parametrize("hw", [(1, 1), (1, 300), (300, 1), (2, 2), (255, 31), (256, 32), (257, 33), (17, 255),
                                (65, 256), (31, 257), (300, 16), (300, 17), (15, 300)])
def test_sizes_around_the_launch_boundaries(hw):
    p, t = _masks((2, 2, *hw), sum(hw), 0.1).long(), _masks((2, 2, *hw), sum(hw) + 1, 0.1).long()
    _check(p, t, 2, include_background=True)
    _check(p, t, 2, include_background=True, distance_metric="taxicab", spacing=[3, 1], directed=True)


def test_height_above_65535():
    rng = np.random.default_rng(11)
    p = torch.from_numpy(rng.random((1, 1, 70000, 3)) < 0.5)
    t = torch.zeros(1, 1, 70000, 3, dtype=torch.bool)
    t[0, 0, 69990:, :2] = True
    t[0, 0, 3, 2] = True
    _check(p, t, 1)
    _check(p, t, 1, distance_metric="chessboard", spacing=[0.5, 2], directed=True)


def test_opposite_corners_round_like_float32():
    p = torch.zeros(1, 1, 5000, 5000, dtype=torch.bool)
    t = torch.zeros_like(p)
    p[0, 0, 0, 0] = t[0, 0, 4999, 4999] = True
    assert 2 * 4999 ** 2 > 1 << 24 and float(np.float32(2 * 4999 ** 2)) != 2 * 4999 ** 2
    _check(p, t, 1)
    _check(p, t, 1, spacing=[0.7, 1.3], distance_metric="taxicab")


def test_edges_use_the_four_axis_neighbours():
    """The centre of a 3 x 3 block without one corner is not an edge: its four axis neighbours are in the mask, only a
    diagonal one is outside (the reference's erosion uses the connectivity-1 cross)."""
    t = torch.zeros(1, 1, 7, 7, dtype=torch.bool)
    t[0, 0, 2:5, 2:5] = True
    t[0, 0, 2, 2] = False
    p = torch.zeros_like(t)
    p[0, 0, 3, 3] = True
    assert _run(p, t, 1, directed=True).item() == 1.0
    _check(p, t, 1, directed=True)
    _check(t, p, 1, distance_metric="taxicab")


def test_all_foreground_and_checkerboard_against_a_corner_blob():
    full = torch.ones(1, 1, 96, 96, dtype=torch.bool)
    holed = full.clone()
    holed[0, 0, 40:50, 40:50] = False
    _check(full, holed, 1)
    _check(full, full, 1)
    i, j = torch.meshgrid(torch.arange(128), torch.arange(128), indexing="ij")
    board = ((i + j) % 2 == 0)[None, None]
    blob = torch.zeros_like(board)
    blob[..., :10, :10] = True
    for metric in hc.METRICS:
        _check(board, blob, 1, distance_metric=metric)


def test_more_pairs_than_one_scratch_launch(monkeypatch):
    p, t = _masks((5, 4, 40, 30), 21).long(), _masks((5, 4, 40, 30), 22).long()
    want = _want(p, t, 4)
    per_pair = _native.lib().mb200_hausdorff_scratch_bytes(40, 30, 0, 1)
    monkeypatch.setattr(_native, "HAUSDORFF_SCRATCH_BYTES", 3 * per_pair)  # 15 pairs in launches of 3
    assert torch.equal(_run(p, t, 4), want)


def test_equal_to_the_reference_op_chain_on_the_same_gpu():
    """On CUDA tensors the reference's own float32 arithmetic (sqrt included) gives the same bits as K19."""
    rng = np.random.default_rng(13)
    for metric in hc.METRICS:
        for spacing in hc.SPACINGS:
            p, t = rng.random((40, 40)) < 0.2, rng.random((40, 40)) < 0.2
            pd, td = torch.from_numpy(p).to(DEV), torch.from_numpy(t).to(DEV)
            want = oh.chain_pair(pd, td, spacing or [1, 1], metric, False).cpu()
            got = _run(pd[None, None], td[None, None], 1, distance_metric=metric, spacing=spacing)
            assert torch.equal(got.reshape(()), want.reshape(())), (metric, spacing)


def test_two_runs_give_identical_bits():
    p, t = _masks((4, 3, 120, 90), 31).long(), _masks((4, 3, 120, 90), 32).long()
    a = _run(p, t, 3, spacing=[0.7, 1.3])
    b = _run(p, t, 3, spacing=[0.7, 1.3])
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_errors_follow_the_reference_order_on_the_gpu():
    from metrics_b200.functional.segmentation import hausdorff_distance

    ok = torch.ones(2, 3, 6, 6, dtype=torch.int64)
    ok[:, :, 2:4, 2:4] = 0
    early_nb, late_empty = ok.clone(), ok.clone()
    early_nb[0, 1, 0, 0] = 2
    early_nb[1, 2] = late_empty[1, 2] = 0
    with pytest.raises(ValueError, match="binarized"):
        hausdorff_distance(early_nb.to(DEV), late_empty.to(DEV), 3)
    empty, late_nb = ok.clone(), ok.clone()
    empty[0, 2] = late_nb[0, 2] = 0
    late_nb[1, 1, 3, 3] = 3
    with pytest.raises(RuntimeError, match="numel"):
        hausdorff_distance(empty.to(DEV), late_nb.to(DEV), 3)
    lab = torch.randint(0, 3, (2, 6, 6))
    with pytest.raises(RuntimeError, match="smaller than num_classes"):
        hausdorff_distance(lab.to(DEV), (lab + 1).to(DEV), 3, input_format="index")
    with pytest.raises(NotImplementedError, match='"bitwise_or_cuda" not implemented for \'Float\''):
        hausdorff_distance(ok.float().to(DEV), ok.to(DEV), 3)
