"""CPU: the COCO mAP oracle against the known answers the reference tree holds (parity PARTIALLY pinned, see
oracle/coco_map.py header): docstring / unit-test constants exactly, and the reference's legacy in-tree evaluator on
crowd-free data — recall statistics to 1e-6, precision statistics loosely (the legacy code compares recall levels in
fp32, COCOeval in fp64, which moves samples at recall levels like 3/10 vs float32(0.3))."""
import numpy as np
import pytest

from oracle.coco_map import coco_evaluate, default_iou_thresholds, default_rec_thresholds
from tests.helpers import LEGACY_MAP_CASES, det_to_numpy, synth_detection


def test_threshold_defaults_are_float32_rounded_doubles():
    thr = default_iou_thresholds()
    assert thr[0] == 0.5 and thr[5] == 0.75 and thr[1] == 0.550000011920929 and thr[-1] == 0.949999988079071
    rec = default_rec_thresholds()
    assert len(rec) == 101 and rec[1] == 0.009999999776482582 and rec[55] == 0.550000011920929 and rec[100] == 1.0


def test_docstring_example():
    """detection/mean_ap.py:250-283"""
    r = coco_evaluate([np.array([[258.0, 41.0, 606.0, 285.0]])], [np.array([0.536])], [np.array([0])],
                      [np.array([[214.0, 41.0, 562.0, 285.0]])], [np.array([0])])
    want = dict(map=0.6, map_50=1.0, map_75=1.0, map_small=-1.0, map_medium=-1.0, map_large=0.6, mar_1=0.6, mar_10=0.6,
                mar_100=0.6, mar_small=-1.0, mar_medium=-1.0, mar_large=0.6)
    for k, v in want.items():
        assert float(r[k]) == pytest.approx(v, abs=1e-7), k
    assert r["classes"].tolist() == [0]


@pytest.mark.parametrize("fmt,expected", [("xyxy", 1.0), ("xywh", 0.0), ("cxcywh", 0.0)])
def test_box_format(fmt, expected):
    """tests/unittests/detection/test_map.py:751-777"""
    r = coco_evaluate([np.array([[0.5, 0.5, 1.0, 1.0]])], [np.array([1.0])], [np.array([0])],
                      [np.array([[0.0, 0.0, 1.0, 1.0]])], [np.array([0])], box_format=fmt, iou_thresholds=[0.2])
    assert float(r["map"]) == expected


def test_missing_50_75_thresholds_and_empty_sides():
    """test_map.py:570-582 (map_50 == map_75 == -1 when not requested) and :479-555 (empty preds / gts do not crash)"""
    box = np.array([[214.15, 41.29, 562.41, 285.07]])
    r = coco_evaluate([box], [np.array([0.5])], [np.array([4])], [box], [np.array([4])], iou_thresholds=[0.1, 0.2])
    assert float(r["map_50"]) == -1.0 and float(r["map_75"]) == -1.0 and float(r["map"]) == 1.0
    r = coco_evaluate([np.zeros((0, 4))], [np.zeros(0)], [np.zeros(0, np.int64)], [box], [np.array([4])])
    assert float(r["map"]) == 0.0 and float(r["mar_100"]) == 0.0  # a class with ground truth but no detection scores 0
    r = coco_evaluate([box], [np.array([0.5])], [np.array([4])], [np.zeros((0, 4))], [np.zeros(0, np.int64)])
    assert float(r["map"]) == -1.0  # no ground truth at all: undefined


@pytest.mark.parametrize("name", list(LEGACY_MAP_CASES))
def test_against_legacy_in_tree_evaluator(golden_det, name):
    preds, target = synth_detection(**LEGACY_MAP_CASES[name])
    r = coco_evaluate(**det_to_numpy(preds, target))
    for k in ("mar_1", "mar_10", "mar_100"):
        np.testing.assert_allclose(r[k], golden_det[f"legacy/{name}/{k}"], rtol=1e-6)
    np.testing.assert_allclose(r["mar_100_per_class_values"], golden_det[f"legacy/{name}/mar_100_per_class"], rtol=1e-6)
    # precision statistics: the legacy evaluator compares recall levels in fp32 (COCOeval: fp64) and sorts with an
    # unstable sort, so ties in scores ("dup") or recall levels sitting on a threshold move a few samples
    for k in ("map", "map_50", "map_75"):
        np.testing.assert_allclose(r[k], golden_det[f"legacy/{name}/{k}"], rtol=2e-2 if name == "dup" else 3e-4)


def test_segm_docstring_known_answer():
    """detection/mean_ap.py:285-340 — the reference's only pinned `iou_type="segm"` value: a 4-pixel prediction and a 4-pixel
    ground truth sharing 3 pixels (IoU 3/5) match at the IoU thresholds 0.5 and 0.55 -> map = mar = 0.2, map_50 1, map_75 0,
    everything "small"."""
    import numpy as np

    from oracle.coco_map import mask_iou

    mask_pred = np.array([[[0, 0, 0, 0, 0], [0, 0, 1, 1, 0], [0, 0, 1, 1, 0], [0, 0, 0, 0, 0], [0, 0, 0, 0, 0]]], bool)
    mask_tgt = np.array([[[0, 0, 0, 0, 0], [0, 0, 1, 0, 0], [0, 0, 1, 1, 0], [0, 0, 1, 0, 0], [0, 0, 0, 0, 0]]], bool)
    assert mask_iou(mask_pred, mask_tgt, np.zeros(1)).tolist() == [[0.6]]
    assert mask_iou(mask_pred, mask_tgt, np.ones(1)).tolist() == [[0.75]]  # crowd: union = the detection's area
    assert mask_iou(mask_pred, np.zeros_like(mask_tgt), np.zeros(1)).tolist() == [[0.0]]
    r = coco_evaluate(None, [np.array([0.536])], [np.array([0])], None, [np.array([0])], det_masks=[mask_pred],
                      gt_masks=[mask_tgt], iou_type="segm")
    want = dict(map=0.2, map_50=1.0, map_75=0.0, map_large=-1.0, map_medium=-1.0, map_small=0.2, mar_1=0.2, mar_10=0.2,
                mar_100=0.2, mar_large=-1.0, mar_medium=-1.0, mar_small=0.2)
    for k, v in want.items():
        assert abs(float(r[k]) - v) < 1e-6, k


# ---- the record-level restatement (match_records / accumulate_records) against COCOeval restated per image -------------
def _legacy_flat_case(name):
    from oracle.coco_map import box_convert_to_xywh
    from tests.coco_map_cases import make_case

    preds, target = synth_detection(**LEGACY_MAP_CASES[name])
    kw = det_to_numpy(preds, target)
    images = []
    for i in range(len(kw["det_labels"])):
        db, gb = box_convert_to_xywh(kw["det_boxes"][i], "xyxy"), box_convert_to_xywh(kw["gt_boxes"][i], "xyxy")
        det = [tuple(b) + (s, lab) for b, s, lab in zip(db.tolist(), kw["det_scores"][i].tolist(), kw["det_labels"][i].tolist())]
        gt = [tuple(b) + (lab, 0, 0.0) for b, lab in zip(gb.tolist(), kw["gt_labels"][i].tolist())]
        images.append(dict(det=det, gt=gt))
    return make_case(images)


def _hand_built(name):
    from tests.coco_map_cases import HAND_BUILT

    return HAND_BUILT[name]()


def _records_equal_coco_evaluate(case):
    from oracle.coco_map import accumulate_records
    from tests.coco_map_cases import coco_eval, oracle_records

    cat, rank, match, ignore, npig = oracle_records(case)
    got = accumulate_records(cat, case["det_score"], rank, match, ignore, npig, npig.shape[0], 0, npig.shape[0],
                             len(case["iou_thr"]), case["rec_thr"], case["max_dets"])
    want = coco_eval(case)
    for name, g in zip(("precision", "recall", "scores"), got):
        np.testing.assert_array_equal(g, want[name], err_msg=name)


@pytest.mark.parametrize("name", list(LEGACY_MAP_CASES))
def test_records_equal_coco_evaluate_legacy(name):
    _records_equal_coco_evaluate(_legacy_flat_case(name))


@pytest.mark.parametrize("name", ["iou_at_threshold", "equal_iou_ties", "crowd_reuse", "area_bounds", "degenerate_boxes",
                                  "label_values", "label_values_micro", "tied_scores", "signed_zero_inf_scores", "mask_edges",
                                  "mask_edges_micro"])
def test_records_equal_coco_evaluate_hand_built(name):
    _records_equal_coco_evaluate(_hand_built(name))


def test_records_equal_coco_evaluate_nan_scores():
    _records_equal_coco_evaluate(_hand_built("nan_scores"))


def _order_key_rank(score, cat):
    """csrc/cocomap.cu's per-image rank restated: coco_det_order_key (NaN -> all ones, else the inverted order key with
    -0 -> +0), rank = number of same-class detections with a smaller key, or an equal key and a smaller index."""
    bits = np.asarray(score, np.float32).view(np.uint32).astype(np.uint64)
    bits = np.where(bits == 0x80000000, 0, bits)
    key = np.where(bits & 0x80000000, ~bits & 0xFFFFFFFF, bits | 0x80000000)  # f32_order_key
    key = np.where(np.isnan(score), 0xFFFFFFFF, ~key & 0xFFFFFFFF)
    idx = np.arange(len(key))
    before = (cat[None, :] == cat[:, None]) & ((key[None, :] < key[:, None]) | ((key[None, :] == key[:, None]) & (idx[None, :] < idx[:, None])))
    return before.sum(1)


@pytest.mark.parametrize("scores", [
    [0.3, float("nan"), 0.9, 0.9],
    [float("nan"), float("-inf"), float("nan"), 0.1, float("inf"), -0.0, 0.0, float("nan"), -1e-45, 1e-45],
    [-0.0, 0.0, -0.0, 0.0, float("inf"), float("-inf")],
])
def test_nan_signed_zero_inf_follow_mergesort_order(scores):
    """The kernel's order key ranks detections exactly as COCOeval's `argsort(-score, kind="mergesort")`: NaN last in input
    order, +-0 tied, -inf just before NaN; match_records writes those ranks."""
    from oracle.coco_map import match_records

    s = np.array(scores, np.float32)
    want = np.empty(len(s), np.int64)
    want[np.argsort(-s, kind="mergesort")] = np.arange(len(s))
    np.testing.assert_array_equal(_order_key_rank(s, np.zeros(len(s), np.int64)), want)
    n = len(s)
    box = np.tile(np.array([[0, 0, 10, 10]], np.float32), (n, 1))
    _, rank, _, _, _ = match_records(box, s, np.zeros(n, np.int64), [n], box[:1], np.zeros(1, np.int64), np.zeros(1, np.uint8),
                                     np.zeros(1), [1], np.array([0]), [0.5], 100)
    np.testing.assert_array_equal(rank, want)


def test_bb_iou_vectorised_equals_scalar_loop():
    from oracle.coco_map import bb_iou, bb_iou_scalar

    rng = np.random.default_rng(0)
    d = np.concatenate([rng.integers(-5, 40, (60, 4)).astype(np.float32), (rng.random((60, 4)) * 50 - 5).astype(np.float32)])
    g = np.concatenate([rng.integers(-5, 40, (30, 4)).astype(np.float32), (rng.random((30, 4)) * 50 - 5).astype(np.float32)])
    crowd = rng.random(60) < 0.3
    got, want = bb_iou(d, g, crowd), bb_iou_scalar(d, g, crowd)
    assert got.tobytes() == want.tobytes()
