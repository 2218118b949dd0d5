"""CPU: the `ious` entry of MeanAveragePrecision's extended summary (reference detection/mean_ap.py:552-555 = pycocotools
COCOeval.computeIoU per (image, category)).  `_pairwise_ious` is plain batched tensor algebra, so it runs on CPU tensors here
and is compared with the per-pair restatement in oracle/coco_map.py::compute_ious; the GPU tests call it through `compute()`."""
import numpy as np
import pytest
import torch

from metrics_b200.detection.mean_ap import MeanAveragePrecision, _pairwise_ious
from oracle.coco_map import box_convert_to_xywh, compute_ious
from tests.helpers import synth_detection


def _state(preds, target, micro=False):
    metric = MeanAveragePrecision(box_format="xyxy", average="micro" if micro else "macro")
    metric.warn_on_many_detections = False
    metric.update(preds, target)
    cat = metric._cat_or_empty
    cpu = torch.device("cpu")
    return dict(
        det_box=cat(metric.detection_box, (0, 4), torch.float32, cpu), det_score=cat(metric.detection_scores, (0,), torch.float32, cpu),
        det_label=cat(metric.detection_labels, (0,), torch.int64, cpu), det_counts=[int(t.shape[0]) for t in metric.detection_labels],
        gt_box=cat(metric.groundtruth_box, (0, 4), torch.float32, cpu), gt_label=cat(metric.groundtruth_labels, (0,), torch.int64, cpu),
        gt_crowd=cat(metric.groundtruth_crowds, (0,), torch.uint8, cpu), gt_counts=[int(t.shape[0]) for t in metric.groundtruth_labels],
        classes=metric._get_classes(), micro=micro,
    )


def _oracle(preds, target, classes, max_det, micro=False):
    zeros = lambda t: np.zeros_like(t)  # noqa: E731
    det_labels = [p["labels"].numpy() for p in preds]
    gt_labels = [t["labels"].numpy() for t in target]
    if micro:
        det_labels, gt_labels, classes = [zeros(x) for x in det_labels], [zeros(x) for x in gt_labels], [0]
    return compute_ious(
        [box_convert_to_xywh(p["boxes"].numpy(), "xyxy") for p in preds], [p["scores"].numpy() for p in preds], det_labels,
        [box_convert_to_xywh(t["boxes"].numpy(), "xyxy") for t in target], gt_labels,
        [t.get("iscrowd", torch.zeros_like(t["labels"])).numpy() for t in target], classes, max_det)


def _same(got, want):
    assert list(got) == list(want)
    blocks = 0
    for key, ref in want.items():
        if isinstance(ref, list):
            assert got[key] == [], key
        else:
            assert tuple(got[key].shape) == ref.shape and got[key].dtype == torch.float32, key
            np.testing.assert_array_equal(got[key].numpy(), ref, err_msg=str(key))  # same fp64 formula -> same float32
            blocks += 1
    return blocks


@pytest.mark.parametrize("max_det", [100, 3])
@pytest.mark.parametrize("micro", [False, True])
def test_against_per_pair_restatement(micro, max_det):
    preds, target = synth_detection(seed=21, n_img=17, n_gt=7, n_det=23, n_cls=5, crowd_frac=0.3, dup_scores=True)
    st = _state(preds, target, micro)
    got = _pairwise_ious(max_det=max_det, **st)
    assert _same(got, _oracle(preds, target, st["classes"], max_det, micro)) > 10
    assert len(got) == 17 * (1 if micro else len(st["classes"]))


def test_empty_images_missing_classes_and_label_gaps():
    box = lambda *rows: torch.tensor(rows, dtype=torch.float32).reshape(-1, 4)  # noqa: E731
    preds = [
        {"boxes": box([0, 0, 10, 10], [5, 5, 15, 15], [0, 0, 4, 4]), "scores": torch.tensor([0.2, 0.9, 0.9]), "labels": torch.tensor([7, 7, 2])},
        {"boxes": box(), "scores": torch.zeros(0), "labels": torch.zeros(0, dtype=torch.long)},
        {"boxes": box([1, 1, 3, 3]), "scores": torch.tensor([0.5]), "labels": torch.tensor([40])},
    ]
    target = [
        {"boxes": box([0, 0, 10, 10], [100, 100, 110, 110]), "labels": torch.tensor([7, 7]), "iscrowd": torch.tensor([0, 1])},
        {"boxes": box([0, 0, 1, 1]), "labels": torch.tensor([2]), "iscrowd": torch.tensor([0])},
        {"boxes": box(), "labels": torch.zeros(0, dtype=torch.long), "iscrowd": torch.zeros(0, dtype=torch.long)},
    ]
    st = _state(preds, target)
    assert st["classes"] == [2, 7, 40]
    got = _pairwise_ious(max_det=100, **st)
    _same(got, _oracle(preds, target, st["classes"], 100))
    assert got[(0, 7)].tolist() == [[pytest.approx(25 / 175), 0.0], [1.0, 0.0]]  # score 0.9 first, then 0.2
    assert got[(0, 2)] == [] and got[(1, 2)] == [] and got[(2, 40)] == [] and got[(1, 7)] == []
    none = _state([preds[1]], [target[2]])
    assert _pairwise_ious(max_det=100, **none) == {}


def test_crowd_union_is_the_detection_area():
    preds = [{"boxes": torch.tensor([[0.0, 0.0, 2.0, 2.0]]), "scores": torch.tensor([0.9]), "labels": torch.tensor([1])}]
    target = [{"boxes": torch.tensor([[0.0, 0.0, 10.0, 1.0], [0.0, 0.0, 10.0, 1.0]]), "labels": torch.tensor([1, 1]),
               "iscrowd": torch.tensor([1, 0])}]
    got = _pairwise_ious(max_det=100, **_state(preds, target))
    assert got[(0, 1)].tolist() == [[pytest.approx(2 / 4), pytest.approx(2 / 12)]]


@pytest.mark.parametrize("device", ["cpu", pytest.param("cuda:0", marks=pytest.mark.gpu)])
def test_detection_order_nan_signed_zero_inf(device):
    """Rows follow COCOeval's `argsort(-score, kind="mergesort")`: NaN last in input order, -0.0 and +0.0 tied in input
    order, +-inf at the ends; the max_det cut keeps the first rows of that order."""
    nan, inf = float("nan"), float("inf")
    scores = [0.3, nan, 0.9, 0.9, -0.0, 0.0, -inf, inf, -0.0, nan, 0.0]
    n = len(scores)
    det_box = torch.tensor([[float(i), 0.0, 10.0, 10.0] for i in range(n)])
    gt_box = torch.tensor([[0.0, 0.0, 10.0, 10.0], [3.0, 0.0, 10.0, 10.0]])
    dev = torch.device(device)
    for max_det in (100, 7, 2):
        got = _pairwise_ious(det_box.to(dev), torch.tensor(scores).to(dev), torch.zeros(n, dtype=torch.int64, device=dev), [n],
                             gt_box.to(dev), torch.zeros(2, dtype=torch.int64, device=dev), torch.zeros(2, dtype=torch.uint8, device=dev),
                             [2], [0], False, max_det)
        want = compute_ious([det_box.numpy()], [np.array(scores, np.float32)], [np.zeros(n, np.int64)], [gt_box.numpy()],
                            [np.zeros(2, np.int64)], [np.zeros(2, np.int64)], [0], max_det)
        got = {k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in got.items()}
        assert _same(got, want) == 1
