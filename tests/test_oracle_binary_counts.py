"""CPU: oracle/binary_counts.py (the reference's stat-score chain restated in torch) against goldens from the unmodified
reference (tests/golden/make_golden_binary_counts.py): every dtype, probabilities and logits, binary and multilabel,
global and samplewise, `ignore_index` in {None, -1, 0}, scores on the dtype-rounded threshold and its neighbours."""
import os

import numpy as np
import pytest
import torch

from oracle import binary_counts as ob
from tests.conftest import GOLDEN_DIR

DTYPES = {0: torch.float32, 1: torch.float16, 2: torch.bfloat16, 3: torch.float64}


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN_DIR, "binary_counts.npz"), allow_pickle=False)


def sets(g):
    for i in range(int(g["n_sets"])):
        key = f"set{i}"
        code, logits, multilabel = (int(v) for v in g[f"{key}/meta"])
        preds = torch.from_numpy(g[f"{key}/preds"]).to(DTYPES[code])
        yield key, preds, bool(logits), bool(multilabel), float(g[f"{key}/threshold"])


def test_oracle_matches_every_golden(golden):
    n = 0
    for key, preds, _, multilabel, thr in sets(golden):
        for ign in (None, -1, 0):
            target = torch.from_numpy(golden[f"{key}/target_ign" if ign == -1 else f"{key}/target"]).long()
            for mda in ("global", "samplewise"):
                got = ob.stat_counts(preds, target, thr, ign, multilabel, mda == "samplewise")
                np.testing.assert_array_equal(got.numpy(), golden[f"{key}/ign{ign}/{mda}"], err_msg=f"{key} {ign} {mda}")
                n += 1
    assert n == 6 * int(golden["n_sets"]) > 1000


def test_goldens_pin_the_dtype_rounded_threshold(golden):
    """A half-precision score is compared with the threshold rounded to its dtype, not with float32(threshold): the goldens
    tell the two rules apart at the thresholds that are not representable in half precision."""
    differs = set()
    for key, preds, logits, multilabel, thr in sets(golden):
        if preds.dtype not in (torch.float16, torch.bfloat16):
            continue
        target = torch.from_numpy(golden[f"{key}/target"]).long()
        s = torch.sigmoid(preds) if logits else preds
        # the float32-threshold rule: widen the (sigmoid of the) score to float32 before comparing
        f32_rule = ob.stat_counts(s.float(), target, thr, None, multilabel, False, logits=False)
        if not np.array_equal(f32_rule.numpy(), golden[f"{key}/ignNone/global"]):
            differs.add((preds.dtype, thr, logits))
    for dtype in (torch.float16, torch.bfloat16):
        for thr in (0.3, 0.9999):
            assert (dtype, thr, False) in differs, (dtype, thr)
    assert (torch.bfloat16, 0.3, True) in differs


def test_vote_ignores_nan():
    """The device branch of the logits vote: a NaN score is neither below 0 nor above 1."""
    x = torch.tensor([float("nan"), 0.2, 0.9])
    assert not ob.is_logits(x)
    assert ob.is_logits(torch.tensor([float("nan"), 1.5]))
    counts = ob.stat_counts(x, torch.tensor([1, 0, 1]), 0.5)
    assert counts.tolist() == [[1, 0, 1, 1]]
