"""CPU: oracle/multiclass_counts.py (the reference's multiclass counting chain restated in torch) against goldens from the
unmodified reference (tests/golden/make_golden_multiclass_counts.py): every target dtype, `ignore_index` in {None, -1, 0,
C - 1, C} and the values ATen wraps to the target's dtype, confusion matrix and stat scores (micro, none, top-2,
samplewise), scores with NaN, +-inf, -0 / +0 and tied maxima."""
import os

import numpy as np
import pytest
import torch

from oracle import multiclass_counts as om
from tests.conftest import GOLDEN_DIR

PREDS = {0: torch.float32, 1: torch.float16, 2: torch.bfloat16, 3: torch.float64}


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN_DIR, "multiclass_counts.npz"), allow_pickle=False)


def sets(g):
    for i in range(int(g["n_sets"])):
        key = f"set{i}"
        code, c, has_ign, ign = (int(v) for v in g[f"{key}/meta"])
        dt = PREDS[code]
        yield (key, torch.from_numpy(g[f"{key}/preds"]).to(dt), torch.from_numpy(g[f"{key}/preds_topk"]).to(dt),
               torch.from_numpy(g[f"{key}/target"]), c, ign if has_ign else None)


def test_oracle_matches_every_golden(golden):
    n = 0
    dtypes = set()
    for key, p, pk, t, c, ign in sets(golden):
        dtypes.add(t.dtype)
        msg = f"{key} {t.dtype} C={c} ignore_index={ign}"
        np.testing.assert_array_equal(om.confusion_matrix(p, t, c, ign).numpy(), golden[f"{key}/confmat"], err_msg=msg)
        lab = torch.from_numpy(golden[f"{key}/labels"])
        np.testing.assert_array_equal(om.confusion_matrix(lab, t, c, ign).numpy(), golden[f"{key}/confmat_labels"], msg)
        for avg in ("micro", "none"):
            got = om.stat_scores(p, t, c, 1, avg, "global", ign)
            np.testing.assert_array_equal(got.T.numpy() if avg == "none" else got.numpy(), golden[f"{key}/stats_{avg}"], msg)
        sw = om.stat_scores(p, t, c, 1, "none", "samplewise", ign)
        np.testing.assert_array_equal(sw.permute(1, 2, 0).numpy(), golden[f"{key}/stats_samplewise"], err_msg=msg)
        if c >= 3:
            tk = t.flatten()
            want = golden[f"{key}/stats_top2"]
            np.testing.assert_array_equal(om.stat_scores(pk, tk, c, 2, "none", "global", ign).T.numpy(), want, msg)
            if not bool(om.topk_tie_rows(pk, 2).any()):  # no row whose order torch.topk leaves open
                np.testing.assert_array_equal(om.stat_scores_topk(pk, tk, c, 2, ign).T.numpy(), want, msg)
        n += 1
    assert dtypes == {torch.int8, torch.uint8, torch.int16, torch.int32, torch.int64, torch.bool}
    assert n == int(golden["n_sets"]) >= 40


def test_goldens_pin_the_wrapped_ignore_index(golden):
    """The reference compares `target != ignore_index` in the target's dtype: uint8 257 drops class 1, -100 drops 156 and -1
    drops 255; int8 255 and int16 65535 drop -1.  The unwrapped comparison would count those rows (or, out of range,
    break the bincount); the goldens tell the two apart, and validate_args=True accepts the wrapped values."""
    seen = set()
    for key, p, _, t, c, ign in sets(golden):
        if ign is None or 0 <= ign <= c or (ign == -1 and t.dtype != torch.uint8):
            continue
        wrapped = torch.tensor(ign).to(t.dtype).item()
        assert wrapped != ign
        dropped = t == wrapped
        assert bool(dropped.any()), key
        want = om.confusion_matrix(p.argmax(1)[~dropped], t[~dropped].long(), c)
        np.testing.assert_array_equal(golden[f"{key}/confmat"], want.numpy(), err_msg=key)
        assert int(golden[f"{key}/validate_raises"]) == 0, key
        seen.add((t.dtype, ign))
    assert seen == {(torch.uint8, 257), (torch.uint8, -100), (torch.uint8, -1), (torch.int8, 255), (torch.int16, 65535)}


def test_topk_lowest_index_rule():
    """The helper for tied top-k rows: equal scores rank by lower column; NaN ranks first; -0 == +0."""
    nan, inf = float("nan"), float("inf")
    p = torch.tensor([[1.0, 3.0, 3.0, 0.0],    # top-1 tie: column 1 first
                      [2.0, 1.0, 1.0, 1.0],    # 2nd/3rd tie at k = 2: column 1 is in, 2 and 3 are out
                      [nan, inf, nan, 0.0],    # NaNs rank first, lower column first
                      [-0.0, 0.0, -1.0, -2.0]])
    assert om.topk_tie_rows(p, 2).tolist() == [True, True, True, True]
    assert om.topk_refined_lowest_index(p, torch.tensor([2, 2, 2, 1]), 2).tolist() == [2, 0, 2, 1]
    assert om.topk_refined_lowest_index(p, torch.tensor([3, 1, 1, 2]), 2).tolist() == [1, 1, 0, 0]
    assert not bool(om.topk_tie_rows(torch.tensor([[0.0, 1.0, 2.0]]), 2).any())
    # a row without ties: the rule and the chain agree
    q = torch.randn(64, 9, generator=torch.Generator().manual_seed(0))
    t = torch.randint(0, 9, (64,), generator=torch.Generator().manual_seed(1))
    assert torch.equal(om.stat_scores_topk(q, t, 9, 3), om.stat_scores(q, t, 9, 3, "none"))
