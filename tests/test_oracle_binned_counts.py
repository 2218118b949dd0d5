"""CPU: oracle/binned_counts.py (the reference's binned precision-recall-curve state chain restated in torch) against goldens
from the unmodified reference (tests/golden/make_golden_binned_counts.py): binary, multiclass, micro and multilabel updates
on both sides of the reference's size rule, every score dtype and threshold kind, unsorted and duplicated thresholds, and the
multilabel `ignore_index` values 0, 1, -1 and uint8 257."""
import os

import numpy as np
import pytest
import torch

from oracle import binned_counts as ob
from tests.conftest import GOLDEN_DIR

SCORES = {0: torch.float32, 1: torch.float16, 2: torch.bfloat16, 3: torch.float64}
KINDS = ["float16", "bfloat16", "float32", "float64", "int64", "list"]
THR_VALUES = [0.5, 0.1, 0.9999, 0.3, 0.0, 1.0, 0.3, 0.7, 0.33333333, 0.9, 0.2, 1e-40, -0.0, 0.70000001]
INT_VALUES = [1, 0, 0, 2, -1]
C = 10


def thresholds(kind):
    if kind == "list":
        return list(THR_VALUES)
    if kind == "int64":
        return torch.tensor(INT_VALUES, dtype=torch.int64)
    return torch.tensor(THR_VALUES, dtype=torch.float64).to(getattr(torch, kind))


def points():
    return torch.tensor(THR_VALUES + INT_VALUES, dtype=torch.float64)


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN_DIR, "binned_counts.npz"), allow_pickle=False)


def inputs(task, dt, n, seed, tdt=torch.int64, ign=None):
    g = torch.Generator().manual_seed(seed)
    if task == "binary":
        return ob.scores_near(points(), (n,), dt, seed), torch.randint(0, 2, (n,), generator=g)
    if task in ("multiclass", "micro"):
        return ob.scores_near(points(), (n, C), dt, seed), torch.randint(0, C, (n,), generator=g)
    p, t = ob.scores_near(points(), (n, 3), dt, seed), torch.randint(0, 2, (n, 3), generator=g)
    if ign == -1:
        t[::3, 1] = -1
    return p, t.to(tdt)


def run(task, p, t, thr, ign=None):
    if task == "binary":
        return ob.binary(p, t, thr)
    if task == "multilabel":
        return ob.multilabel(p, t, 3, thr, ign)
    return ob.multiclass(p, t, C, thr, None, "micro" if task == "micro" else None)


def sets(g):
    for i in range(int(g["n_sets"])):
        key = f"set{i}"
        code, kind, n, seed, u8, has_ign, ign = (int(v) for v in g[f"{key}/meta"])
        yield key, str(g[f"{key}/task"]), SCORES[code], KINDS[kind], n, seed, bool(u8), ign if has_ign else None


def test_oracle_matches_every_golden(golden):
    seen = set()
    for key, task, dt, kind, n, seed, u8, ign in sets(golden):
        want = golden[f"{key}/state"]
        if u8:
            assert want.size == 0, key  # the reference raised (checked below)
            continue
        p, t = inputs(task, dt, n, seed, torch.int64, ign)
        got = run(task, p, t, thresholds(kind), ign)
        np.testing.assert_array_equal(got.numpy(), want, err_msg=f"{key} {task} {dt} {kind} n={n} ignore_index={ign}")
        seen.add((task, dt, kind))
    assert len(seen) == 4 * 4 * 6


def test_goldens_pin_both_branches_and_their_dtypes(golden):
    """Above the size rule the reference compares in the score dtype, below it in the promoted dtype: for half scores and
    float32 / float64 thresholds the two give different counts on these inputs, and each golden agrees with its own branch
    only.  Below the rule float64 thresholds count a float32 score equal to float32(0.7) (< 0.7) as negative."""
    differ = 0
    for key, task, dt, kind, n, seed, u8, ign in sets(golden):
        if task != "binary" or kind not in ("float32", "float64"):
            continue
        p, t = inputs(task, dt, n, seed)
        thr = thresholds(kind)
        vec, loop = ob.binary_update_vectorized(p, t, thr), ob.binary_update_loop(p, t, thr)
        want = golden[f"{key}/state"]
        mine = loop if n > ob.BINARY_LOOP_ABOVE else vec
        np.testing.assert_array_equal(mine.numpy(), want, err_msg=key)
        if not torch.equal(vec, loop):
            differ += 1
            assert not np.array_equal((vec if mine is loop else loop).numpy(), want), key
    assert differ >= 8  # f16 / bf16 x f32 / f64 on both sizes, and f32 x f64
    x = torch.tensor([0.7], dtype=torch.float32)
    assert ob.binary_update_vectorized(x, torch.tensor([1]), torch.tensor([0.7], dtype=torch.float64))[0, 1, 1] == 0


def test_uint8_multilabel_ignore_index_makes_the_reference_raise(golden):
    """The reference writes -4 * L * T into a uint8 target; it wraps to 196 here and the bincount outgrows its reshape.
    The oracle (and the kernel) drop the entries its mask selects instead: uint8 257 is label 1."""
    n_u8 = 0
    for key, task, dt, kind, n, seed, u8, ign in sets(golden):
        if not u8:
            continue
        n_u8 += 1
        p, t = inputs(task, dt, n, seed, torch.uint8, ign)
        got = ob.multilabel(p, t, 3, thresholds(kind), ign)
        wide = ob.multilabel(p, t.long(), 3, thresholds(kind), 1 if ign == 257 else ign)
        assert torch.equal(got, wide), key
        assert int(got[0].sum()) < 3 * n, key  # something was dropped
    assert n_u8 == 4 * 6 * 3


def test_compare_dtype_rule():
    f16, bf16, f32, f64 = torch.float16, torch.bfloat16, torch.float32, torch.float64
    assert ob.compare_dtype(f16, f32, 50_000) == f32 and ob.compare_dtype(f16, f32, 50_001) == f16
    assert ob.compare_dtype(f16, bf16, 10) == f32 and ob.compare_dtype(bf16, torch.int64, 10) == bf16
    assert ob.compare_dtype(f32, f64, 10_000, 10) == f64 and ob.compare_dtype(f32, f64, 10_001, 10) == f32
    assert ob.compare_dtype(f16, f64, 10**7, 3, multilabel=True) == f64
