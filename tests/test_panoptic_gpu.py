"""GPU: kernel K18 (panoptic quality) — the four states bit-equal to the numpy oracle over every integer dtype pair and
layout, the reference's goldens through both classes and both functionals, unknown categories, the capacity repeat,
run-to-run bits, merge_state, forward() and the state dtypes."""
import numpy as np
import pytest
import torch

from oracle import panoptic as op
from tests import panoptic_cases as pc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = pc.golden_cases()


def _metric(case):
    from metrics_b200.detection import ModifiedPanopticQuality, PanopticQuality

    cls = ModifiedPanopticQuality if case["modified"] else PanopticQuality
    return cls(case["things"], case["stuffs"], **case["kwargs"]).to(DEV)


def _states(m):
    return m.iou_sum, m.true_positives, m.false_positives, m.false_negatives


def _oracle(batches, things, stuffs, modified):
    state = None
    for p, t in batches:
        got = op.update(p.cpu().numpy(), t.cpu().numpy(), things, stuffs, modified)
        state = list(got) if state is None else [a + b for a, b in zip(state, got)]
    return state


def assert_equal_states(got, want):
    for g, w, name in zip(got, want, pc.STATES):
        g = g.cpu().numpy()
        assert g.dtype == np.asarray(w).dtype and np.array_equal(g.view(np.uint8), np.asarray(w).view(np.uint8)), (name, g, w)


@pytest.fixture(scope="module")
def golden():
    return pc.load()


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_goldens_through_the_class(golden, case):
    m = _metric(case)
    pc.assert_output(golden[f"{case['name']}/compute_empty"], m.compute())
    for p, t in case["batches"]:
        m.update(p.to(DEV), t.to(DEV))
    pc.assert_states(golden, case["name"], _states(m))
    pc.assert_output(golden[f"{case['name']}/compute"], m.compute())


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_goldens_through_the_functional(golden, case):
    from metrics_b200.functional.detection import modified_panoptic_quality, panoptic_quality

    fn = modified_panoptic_quality if case["modified"] else panoptic_quality
    p, t = case["batches"][0]
    pc.assert_output(golden[f"{case['name']}/functional"], fn(p.to(DEV), t.to(DEV), case["things"], case["stuffs"], **case["kwargs"]))


@pytest.mark.parametrize("pdt", pc.INT_DTYPES, ids=str)
@pytest.mark.parametrize("tdt", pc.INT_DTYPES, ids=str)
@pytest.mark.parametrize("modified", [False, True])
def test_states_match_the_oracle_for_every_dtype_pair(pdt, tdt, modified):
    g = torch.Generator().manual_seed(hash((str(pdt), str(tdt), modified)) % 10000)
    cats = [0, 1, 2, 3, 4, 5, 6, 9]
    t = pc.blocky(g, (4, 37, 53), cats, 5, block=6)
    p = pc.perturb(g, t, 0.2, cats, 5)
    p, t = p.to(pdt), t.to(tdt)
    m = _metric({"modified": modified, "things": {1, 2, 3}, "stuffs": {4, 5, 6}, "kwargs": {"allow_unknown_preds_category": True}})
    m.update(p.to(DEV), t.to(DEV))
    assert_equal_states(_states(m), _oracle([(p, t)], {1, 2, 3}, {4, 5, 6}, modified))


@pytest.mark.parametrize("shape", [(3, 1, 2), (2, 1000), (2, 4097), (1, 3, 31, 33), (2, 2, 3, 50, 70), (1, 300, 301)])
def test_states_match_the_oracle_at_size_edges(shape):
    g = torch.Generator().manual_seed(sum(shape))
    t = pc.blocky(g, shape, [1, 2, 5, 8], 7, block=3)
    p = pc.perturb(g, t, 0.3, [1, 2, 5, 8], 7)
    for modified in (False, True):
        m = _metric({"modified": modified, "things": {1, 2}, "stuffs": {5}, "kwargs": {"allow_unknown_preds_category": True}})
        m.update(p.to(DEV), t.to(DEV))
        assert_equal_states(_states(m), _oracle([(p, t)], {1, 2}, {5}, modified))


def test_non_contiguous_and_offset_inputs():
    g = torch.Generator().manual_seed(5)
    t = pc.blocky(g, (4, 20, 24), [1, 2, 5], 3)
    p = pc.perturb(g, t, 0.3, [1, 2, 5], 3)
    want = _oracle([(p[:, ::2], t[:, ::2])], {1, 2}, {5}, False)
    m = _metric({"modified": False, "things": {1, 2}, "stuffs": {5}, "kwargs": {}})
    m.update(p.to(DEV)[:, ::2], t.to(DEV)[:, ::2])
    assert_equal_states(_states(m), want)
    # a view starting one element into its storage: not aligned to a (category, instance) pair
    flat_p, flat_t = p.to(DEV).reshape(-1), t.to(DEV).reshape(-1)
    bp = torch.empty(flat_p.numel() + 1, dtype=p.dtype, device=DEV)
    bt = torch.empty_like(bp)
    bp[1:], bt[1:] = flat_p, flat_t
    m = _metric({"modified": False, "things": {1, 2}, "stuffs": {5}, "kwargs": {}})
    m.update(bp[1:].view(p.shape), bt[1:].view(t.shape))
    assert_equal_states(_states(m), _oracle([(p, t)], {1, 2}, {5}, False))


def test_unknown_preds_raise_and_leave_the_states_unchanged():
    from metrics_b200.detection import PanopticQuality

    p0, t0 = pc.inputs0()
    p1, t1 = pc.inputs1()
    m = PanopticQuality({0, 1}, {6, 7}).to(DEV)
    m.update(p0.to(DEV), t0.to(DEV))
    before = [s.clone() for s in _states(m)]
    with pytest.raises(ValueError) as info:
        m.update(p1.to(DEV), t1.to(DEV))
    flat = p1.flatten(1, -2)
    assert str(info.value) == f"Unknown categories found: {flat[flat[..., 0] == 10].to(DEV)}"
    assert all(torch.equal(a, b) for a, b in zip(before, _states(m)))


def _one_segment_per_pixel(side, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.stack([torch.randint(1, 3, (side, side), generator=g), torch.randperm(side * side, generator=g).view(side, side)], -1)
    p = t.clone()
    p[..., 1] = torch.roll(p[..., 1], 1, 1)
    p[::7, ::5, 1] = t[::7, ::5, 1]
    return p[None], t[None]


@pytest.mark.parametrize("modified", [False, True])
def test_capacity_repeat_one_instance_per_pixel(modified):
    p, t = _one_segment_per_pixel(512, 1)
    m = _metric({"modified": modified, "things": {1, 2}, "stuffs": {}, "kwargs": {}})
    m.update(p.to(DEV), t.to(DEV))
    assert_equal_states(_states(m), _oracle([(p, t)], {1, 2}, set(), modified))
    assert int(m.true_positives.sum()) > 0


def test_capacity_repeat_in_a_mixed_batch():
    g = torch.Generator().manual_seed(3)
    dense_p, dense_t = _one_segment_per_pixel(512, 2)
    t = pc.blocky(g, (3, 512, 512), [1, 2, 5], 4, block=16)
    p = pc.perturb(g, t, 0.05, [1, 2, 5], 4)
    p, t = torch.cat([p[:1], dense_p, p[1:]]), torch.cat([t[:1], dense_t, t[1:]])
    for modified in (False, True):
        m = _metric({"modified": modified, "things": {1, 2}, "stuffs": {5}, "kwargs": {}})
        m.update(p.to(DEV), t.to(DEV))
        assert_equal_states(_states(m), _oracle([(p, t)], {1, 2}, {5}, modified))


def test_areas_above_2_24_use_the_float32_rule():
    """The oracle's result for this case (60 s in numpy): the target segment is a false negative only under the float32
    division rule."""
    for case in pc.oracle_only_cases():
        m = _metric(case)
        p, t = case["batches"][0]
        m.update(p.to(DEV), t.to(DEV))
        want = (np.array([0.0, 1.0]), np.array([0, 1], np.int32), np.array([3, 0], np.int32), np.array([1, 0], np.int32))
        assert_equal_states(_states(m), want)


def test_same_bits_on_two_runs():
    g = torch.Generator().manual_seed(11)
    t = pc.blocky(g, (4, 256, 256), [1, 2, 3, 5, 6], 50, block=5)
    p = pc.perturb(g, t, 0.1, [1, 2, 3, 5, 6], 50)
    runs = []
    for _ in range(2):
        m = _metric({"modified": True, "things": {1, 2, 3}, "stuffs": {5, 6}, "kwargs": {}})
        m.update(p.to(DEV), t.to(DEV))
        runs.append([s.cpu() for s in _states(m)])
    assert all(torch.equal(a, b) for a, b in zip(*runs))
    assert_equal_states(runs[0], _oracle([(p, t)], {1, 2, 3}, {5, 6}, True))


def test_merge_state_of_two_halves_equals_the_whole():
    g = torch.Generator().manual_seed(12)
    t = pc.blocky(g, (6, 40, 48), [1, 2, 5], 4)
    p = pc.perturb(g, t, 0.2, [1, 2, 5], 4)
    case = {"modified": False, "things": {1, 2}, "stuffs": {5}, "kwargs": {}}
    whole, a, b = _metric(case), _metric(case), _metric(case)
    whole.update(p.to(DEV), t.to(DEV))
    a.update(p[:3].to(DEV), t[:3].to(DEV))
    b.update(p[3:].to(DEV), t[3:].to(DEV))
    a.merge_state(b)
    assert all(torch.equal(x, y) for x, y in zip(_states(a), _states(whole)))  # IoU terms above 0.5 add exactly
    assert torch.equal(a.compute(), whole.compute())


def test_forward_returns_the_batch_value_and_accumulates():
    from metrics_b200.detection import PanopticQuality
    from metrics_b200.functional.detection import panoptic_quality

    p0, t0 = pc.inputs0()
    m = PanopticQuality({0, 1}, {6, 7}).to(DEV)
    v1 = m(p0.to(DEV), t0.to(DEV))
    v2 = m(t0.to(DEV), t0.to(DEV))
    assert torch.equal(v1, panoptic_quality(p0.to(DEV), t0.to(DEV), {0, 1}, {6, 7}))
    assert float(v2) == 1.0
    both = _oracle([(p0, t0), (t0, t0)], {0, 1}, {6, 7}, False)
    assert_equal_states(_states(m), both)


def test_state_dtypes_and_device():
    m = _metric({"modified": True, "things": {0, 1}, "stuffs": {2}, "kwargs": {}})
    p, t = pc.inputs0()
    m.update(p.to(DEV) % 3, t.to(DEV) % 3)
    assert m.iou_sum.dtype == torch.float64 and m.iou_sum.is_cuda
    assert all(s.dtype == torch.int32 and s.is_cuda for s in _states(m)[1:])
