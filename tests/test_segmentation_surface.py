"""CPU: the public surface of the segmentation metrics against the reference's (tests/golden/segmentation_surface.json,
dumped by tests/golden/make_golden_segmentation.py), and the host layer — validation, error precedence, the epilogues and
the states — replayed over every golden with the numpy oracle standing in for kernel K15."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import segmentation as osg
from tests import segmentation_cases as sc
from tests.conftest import GOLDEN_DIR
from tests.golden.make_golden_segmentation import seg_states, seg_surface


@pytest.fixture(scope="module")
def ref():
    return json.load(open(os.path.join(GOLDEN_DIR, "segmentation_surface.json")))


def test_surface_matches_the_reference(ref):
    mine = seg_surface("metrics_b200")
    want = dict(ref["surface"])
    want["segmentation.__all__"] = [n for n in want["segmentation.__all__"] if n != "HausdorffDistance"]
    want["functional.segmentation.__all__"] = [n for n in want["functional.segmentation.__all__"] if n != "hausdorff_distance"]
    assert mine == want


def test_state_registry_matches_the_reference(ref):
    assert seg_states("metrics_b200") == ref["states"]


def test_not_exported_from_the_top_level_package():
    import metrics_b200

    assert not hasattr(metrics_b200, "MeanIoU") and not hasattr(metrics_b200, "DiceScore")


def _standin(preds, target, num_classes, index_format, mul, drop_background, err_flag=None):
    """`_native.segmentation_overlap_counts` on CPU tensors, from the numpy oracle (same contract, same flag bits)."""
    if index_format:
        p, t = preds.numpy(), target.numpy()
        flag = 0
        for x, neg, big in ((p, 1, 2), (t, 4, 8)):
            flag |= neg if (x < 0).any() else 0
            flag |= big if (x >= num_classes).any() else 0
        if err_flag is not None:
            err_flag |= flag
        c = num_classes
    else:
        wide = preds.dtype in (torch.bfloat16,)
        p = (preds.float() if wide else preds).contiguous().numpy()
        t = (target.float() if wide else target).contiguous().numpy()
        c = preds.shape[1]
    out = osg.counts(p, t, c, not drop_background, index_format, "mul" if mul else "and")
    dtype = torch.float64 if preds.is_floating_point() else torch.int64
    return torch.stack([torch.from_numpy(np.ascontiguousarray(x)).to(dtype) for x in out])


@pytest.fixture
def host(monkeypatch):
    from metrics_b200 import _native

    monkeypatch.setattr(_native, "segmentation_overlap_counts", _standin)


def test_goldens_through_classes_and_functionals_on_the_standin(host):
    golden = sc.load()
    for key, case in sc.cases(golden):
        sc.check_case(golden, key, case, "cpu")


def test_error_messages_and_precedence(host, ref):
    from metrics_b200 import segmentation as S  # noqa: N812
    from metrics_b200.functional import segmentation as F  # noqa: N812

    errors = ref["errors"]
    lab = torch.randint(0, 4, (2, 5, 5))
    neg, big = lab.clone(), lab.clone()
    neg[0, 1, 1], big[1, 2, 2] = -1, 4
    both = neg.clone()
    both[1, 2, 2] = 4
    calls = {
        "preds_negative": lambda: F.dice_score(neg, lab, 4, input_format="index"),
        "preds_too_large": lambda: F.dice_score(big, lab, 4, input_format="index"),
        "target_negative": lambda: F.dice_score(lab, neg, 4, input_format="index"),
        "target_too_large": lambda: F.dice_score(lab, big, 4, input_format="index"),
        "preds_both": lambda: F.mean_iou(both, big, 4, input_format="index"),
        "preds_large_target_negative": lambda: F.generalized_dice_score(big, neg, 4, input_format="index"),
        "int32_index": lambda: F.dice_score(lab.int(), lab.int(), 4, input_format="index"),
        "float_mean_iou": lambda: F.mean_iou(torch.rand(2, 3, 4, 4), torch.rand(2, 3, 4, 4), 3),
        "shape": lambda: F.dice_score(lab, lab[:1], 4, input_format="index"),
        "dice_2d": lambda: F.dice_score(torch.ones(2, 3, dtype=torch.long), torch.ones(2, 3, dtype=torch.long), 3),
        "num_classes": lambda: S.MeanIoU(0),
        "input_format": lambda: S.DiceScore(3, input_format="x"),
        "average": lambda: S.DiceScore(3, average="samples"),
        "weight_type": lambda: S.GeneralizedDiceScore(3, weight_type="cubic"),
        "per_class": lambda: S.MeanIoU(3, per_class=1),
        "include_background": lambda: S.GeneralizedDiceScore(3, include_background=None),
    }
    assert set(calls) == set(errors)
    for name, call in calls.items():
        kind, msg = errors[name]
        with pytest.raises(Exception) as info:
            call()
        assert type(info.value).__name__ == kind and str(info.value) == msg, (name, info.value)


def test_a_raising_update_leaves_the_states_unchanged(host):
    from metrics_b200.segmentation import GeneralizedDiceScore, MeanIoU

    lab = torch.randint(0, 4, (2, 5, 5))
    bad = lab.clone()
    bad[0, 0, 0] = 9
    for m in (MeanIoU(4, input_format="index"), GeneralizedDiceScore(4, input_format="index")):
        m.update(lab, lab)
        before = {k: v.clone() for k, v in m.metric_state.items()}
        with pytest.raises(RuntimeError, match="smaller than num_classes"):
            m.update(lab, bad)
        assert all(torch.equal(before[k], v) for k, v in m.metric_state.items())
