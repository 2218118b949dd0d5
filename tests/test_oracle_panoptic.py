"""CPU: the panoptic-quality oracle (numpy) and the torch op chain (oracle/panoptic.py) against the reference's goldens
(tests/golden/panoptic.npz), bit for bit, and the division rule both rest on."""
import numpy as np
import pytest
import torch

from oracle import panoptic as op
from tests import panoptic_cases as pc

CASES = pc.golden_cases()


@pytest.fixture(scope="module")
def golden():
    return pc.load()


def _batch_sum(case, update):
    """The reference's state after its updates: each batch summed over its images, then added to the state."""
    state = None
    for p, t in case["batches"]:
        got = update(p, t, case["things"], case["stuffs"], case["modified"])
        got = [torch.as_tensor(np.asarray(x)) if not isinstance(x, torch.Tensor) else x for x in got]
        state = got if state is None else [a + b for a, b in zip(state, got)]
    return state


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_oracle_matches_the_reference(golden, case):
    pc.assert_states(golden, case["name"], _batch_sum(case, lambda p, t, *a: op.update(p.numpy(), t.numpy(), *a)))


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_chain_matches_the_reference(golden, case):
    pc.assert_states(golden, case["name"], _batch_sum(case, op.chain_update))


@pytest.mark.parametrize("case", [c for c in CASES if c["batches"][0][0].numel()], ids=lambda c: c["name"])
def test_oracle_compute_matches_the_reference(golden, case):
    states = _batch_sum(case, lambda p, t, *a: op.update(p.numpy(), t.numpy(), *a))
    pq, sq, rq, pq_avg, sq_avg, rq_avg = op.compute(*states)
    if case["modified"] or not case["kwargs"].get("return_per_class") and not case["kwargs"].get("return_sq_and_rq"):
        pc.assert_output(golden[f"{case['name']}/compute"], pq_avg)


def test_torch_int64_division_is_float32_of_each_operand_then_one_division():
    g = np.random.default_rng(7)
    a = g.integers(1 << 24, 1 << 40, 200_000)
    b = g.integers(1 << 24, 1 << 40, 200_000)
    want = op.f32_ratio(a, b)
    got = (torch.from_numpy(a) / torch.from_numpy(b)).numpy()
    assert got.dtype == np.float32 and np.array_equal(got, want)
    # the example that separates the rule from rounding the exact quotient: exactly 0.5, not a match
    assert op.f32_ratio(16777217, 33554433) == np.float32(0.5)
    assert 16777217 / 33554433 > 0.5  # in float64 it would be one
