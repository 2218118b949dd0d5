"""Oracle for detection.MeanAveragePrecision (bbox, and segm on decoded masks), numpy/fp64.  TEST INFRASTRUCTURE ONLY — see oracle/__init__.py.

PARITY STATUS: **partially pinned**.  In the reference all mAP arithmetic happens inside the third-party package
`pycocotools >2.0.0,<2.1.0` (`cocoeval.py` COCOeval.evaluate/accumulate/summarize and `maskApi.c:bbIou`; call sites
detection/mean_ap.py:538-546), which is NOT under /root/reference and is not installed in any container of this project.
This file restates that published algorithm (function by function, below) together with the reference-side marshalling
that IS in the tree (detection/mean_ap.py:478-519 update, :827-859 box conversion, :867-958 COCO-format dicts, :632-648
stat names).  It is pinned only by the known answers the reference tree itself holds (class docstring
detection/mean_ap.py:250-283; tests/unittests/detection/test_map.py:479-555, :570-582, :751-777) and cross-checked on
crowd-free data against the reference's legacy in-tree evaluator detection/_mean_ap.py for the statistics whose semantics
coincide (see tests/golden/make_golden.py::map_golden).  Beyond those, 1e-6 parity against a real pycocotools is unverified.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np

AREA_RANGES = [(0.0, 1e10), (0.0, 32.0**2), (32.0**2, 96.0**2), (96.0**2, 1e10)]  # all, small, medium, large
EPS = np.spacing(1)


def default_iou_thresholds() -> List[float]:
    """torch.linspace(0.5, 0.95, 10).tolist() (detection/mean_ap.py:411): float32 values widened to double.  torch's
    float32 linspace is NOT the correctly rounded float32 of the exact grid for every index (numpy's is), and a one-ulp
    difference in a recall threshold moves `searchsorted` whenever a recall level k/npig lands on it — so the oracle asks
    torch itself for these constants."""
    import torch

    return torch.linspace(0.5, 0.95, round((0.95 - 0.5) / 0.05) + 1).tolist()


def default_rec_thresholds() -> List[float]:
    """torch.linspace(0, 1, 101).tolist() (detection/mean_ap.py:417); see default_iou_thresholds."""
    import torch

    return torch.linspace(0.0, 1.00, round(1.00 / 0.01) + 1).tolist()


def box_convert_to_xywh(boxes: np.ndarray, fmt: str) -> np.ndarray:
    """torchvision.ops.box_convert(boxes, fmt, "xywh") in float32 (detection/mean_ap.py:846): cxcywh goes through xyxy."""
    b = boxes.astype(np.float32).reshape(-1, 4)
    if fmt == "xywh":
        return b
    if fmt == "cxcywh":
        cx, cy, w, h = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
        half = np.float32(0.5)
        b = np.stack([cx - half * w, cy - half * h, cx + half * w, cy + half * h], axis=1).astype(np.float32)
    x1, y1, x2, y2 = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    return np.stack([x1, y1, x2 - x1, y2 - y1], axis=1).astype(np.float32)


def bb_iou(dt: np.ndarray, gt: np.ndarray, iscrowd: np.ndarray) -> np.ndarray:
    """maskApi.c:bbIou — IoU of xywh boxes in double; for a crowd gt the union is the detection's area.  Vectorised over the
    [D, G] grid in bbIou's operation order: `np.fmin` / `np.fmax` are C's `fmin` / `fmax`, and numpy ufuncs never contract a
    product and a sum into one FMA, so every value is the one the scalar loop (`bb_iou_scalar`) computes."""
    d = dt.astype(np.float64).reshape(-1, 4)
    g = gt.astype(np.float64).reshape(-1, 4)
    dx, dy, dw, dh = (d[:, i:i + 1] for i in range(4))
    gx, gy, gw, gh = (g[None, :, i] for i in range(4))
    w = np.fmin(dx + dw, gx + gw) - np.fmax(dx, gx)
    h = np.fmin(dy + dh, gy + gh) - np.fmax(dy, gy)
    inter = w * h
    da, ga = dw * dh, gw * gh
    union = np.where(np.asarray(iscrowd, bool).reshape(1, -1), da, da + ga - inter)
    with np.errstate(divide="ignore", invalid="ignore"):
        iou = inter / union
    return np.where((w <= 0) | (h <= 0), 0.0, iou)  # `if (w <= 0) continue`: a NaN width is not skipped


def bb_iou_scalar(dt: np.ndarray, gt: np.ndarray, iscrowd: np.ndarray) -> np.ndarray:
    """bb_iou as maskApi.c:bbIou's loop, pair by pair (the check on the vectorised version; NaN-free boxes only)."""
    d = dt.astype(np.float64)
    g = gt.astype(np.float64)
    out = np.zeros((d.shape[0], g.shape[0]), dtype=np.float64)
    for gi in range(g.shape[0]):
        ga = g[gi, 2] * g[gi, 3]
        for di in range(d.shape[0]):
            da = d[di, 2] * d[di, 3]
            w = min(d[di, 0] + d[di, 2], g[gi, 0] + g[gi, 2]) - max(d[di, 0], g[gi, 0])
            if w <= 0:
                continue
            h = min(d[di, 1] + d[di, 3], g[gi, 1] + g[gi, 3]) - max(d[di, 1], g[gi, 1])
            if h <= 0:
                continue
            inter = w * h
            union = da if iscrowd[gi] else da + ga - inter
            out[di, gi] = inter / union
    return out


def compute_ious(det_boxes: Sequence[np.ndarray], det_scores: Sequence[np.ndarray], det_labels: Sequence[np.ndarray],
                 gt_boxes: Sequence[np.ndarray], gt_labels: Sequence[np.ndarray], gt_crowds: Sequence[np.ndarray],
                 classes: Sequence[int], max_det: int) -> dict:
    """COCOeval.computeIoU for every (image, category), i.e. the `ious` entry of the reference's extended summary
    (detection/mean_ap.py:552-555 reads `coco_eval.ious`): detections of the pair sorted by descending score (mergesort),
    cut to the largest maxDets, ground truths in dataset order; `[]` when either side is empty (maskUtils.iou of an empty
    list), else a float32 `[D, G]` array (the reference converts the double matrix with `torch.tensor(x, float32)`)."""
    out = {}
    for img in range(len(det_labels)):
        for cat in classes:
            d_sel = np.nonzero(np.asarray(det_labels[img]).reshape(-1) == cat)[0]
            g_sel = np.nonzero(np.asarray(gt_labels[img]).reshape(-1) == cat)[0]
            if len(d_sel) == 0 or len(g_sel) == 0:
                out[(img, int(cat))] = []
                continue
            order = np.argsort(-np.asarray(det_scores[img], dtype=np.float64).reshape(-1)[d_sel], kind="mergesort")[:max_det]
            d = np.asarray(det_boxes[img]).reshape(-1, 4)[d_sel][order]
            g = np.asarray(gt_boxes[img]).reshape(-1, 4)[g_sel]
            crowd = np.asarray(gt_crowds[img]).reshape(-1)[g_sel]
            out[(img, int(cat))] = bb_iou(d, g, crowd).astype(np.float32)
    return out


def mask_iou(dt: np.ndarray, gt: np.ndarray, iscrowd: np.ndarray) -> np.ndarray:
    """maskApi.c:rleIou on decoded masks (bool [n, H, W]): intersection / union of pixel counts in double; no intersection
    -> 0 (`if(i==0) u=1`); for a crowd gt the union is the detection's area.  (pycocotools walks run-length codes; the counts
    it arrives at are these.)"""
    out = np.zeros((dt.shape[0], gt.shape[0]), dtype=np.float64)
    for gi in range(gt.shape[0]):
        ga = int(gt[gi].sum())
        for di in range(dt.shape[0]):
            inter = int(np.logical_and(dt[di], gt[gi]).sum())
            if inter == 0:
                continue
            da = int(dt[di].sum())
            out[di, gi] = inter / (da if iscrowd[gi] else da + ga - inter)
    return out


def match_detections(ious, gt_crowd, gt_ig, iou_thrs):
    """The greedy matching loop of COCOeval.evaluateImg: `ious` [D, G] with the detections in descending-score order and the
    ground truths with the ignored ones last.  Returns dtm [T, D] (index + 1 of the matched ground truth, 0 = none) and the
    "matched to an ignored ground truth" flags [T, D]."""
    D, G = ious.shape
    T = len(iou_thrs)
    gtm = np.zeros((T, G), dtype=np.int64)
    dtm = np.zeros((T, D), dtype=np.int64)
    dt_ig = np.zeros((T, D), dtype=bool)
    if D and G:
        for ti, t in enumerate(iou_thrs):
            for di in range(D):
                iou = min(t, 1 - 1e-10)
                m = -1
                for gi in range(G):
                    if gtm[ti, gi] > 0 and not gt_crowd[gi]:
                        continue
                    if m > -1 and not gt_ig[m] and gt_ig[gi]:
                        break
                    if ious[di, gi] < iou:
                        continue
                    iou = ious[di, gi]
                    m = gi
                if m == -1:
                    continue
                dt_ig[ti, di] = gt_ig[m]
                dtm[ti, di] = m + 1
                gtm[ti, m] = di + 1
    return dtm, dt_ig


def _evaluate_img(dt_boxes, dt_scores, gt_boxes, gt_crowd, gt_area, iou_thrs, area_rng, max_det, masks=False):
    """COCOeval.computeIoU + evaluateImg for one (image, category, area range).  Returns None when both lists are empty.
    `masks`: dt_boxes / gt_boxes are boolean instance masks [n, H, W] (iouType "segm")."""
    if len(dt_scores) == 0 and len(gt_boxes) == 0:
        return None
    dt_order = np.argsort(-dt_scores, kind="mergesort")[:max_det]
    dt_boxes, dt_scores = dt_boxes[dt_order], dt_scores[dt_order]
    gt_ig = np.array([bool(c) or (a < area_rng[0] or a > area_rng[1]) for c, a in zip(gt_crowd, gt_area)], dtype=bool)
    gt_order = np.argsort(gt_ig, kind="mergesort")
    gt_boxes, gt_crowd, gt_ig = gt_boxes[gt_order], gt_crowd[gt_order], gt_ig[gt_order]
    T, G, D = len(iou_thrs), len(gt_boxes), len(dt_scores)
    ious = (mask_iou if masks else bb_iou)(dt_boxes, gt_boxes, gt_crowd) if D and G else np.zeros((D, G))
    dtm, dt_ig = match_detections(ious, gt_crowd, gt_ig, iou_thrs)
    if masks:  # detection/mean_ap.py:923-924: the detection's "area" is its mask area
        dt_area = dt_boxes.sum(axis=(1, 2)).astype(np.float64) if D else np.zeros(0)
    else:
        dt_area = dt_boxes[:, 2].astype(np.float64) * dt_boxes[:, 3].astype(np.float64) if D else np.zeros(0)
    out_of_range = (dt_area < area_rng[0]) | (dt_area > area_rng[1])
    dt_ig = dt_ig | ((dtm == 0) & out_of_range[None, :])
    return {"dtm": dtm, "dt_ig": dt_ig, "scores": dt_scores, "gt_ig": gt_ig}


def sample_pr_curve(tp, fp, sorted_scores, npig, rec_thrs):
    """The per-threshold tail of COCOeval.accumulate: cumulative TP / FP counts of the score-sorted detections -> (final
    recall, precision envelope sampled at the recall thresholds, the scores at those samples)."""
    R, nd = len(rec_thrs), len(tp)
    rc = tp / npig
    pr = tp / (fp + tp + EPS)
    q = np.zeros(R)
    ss = np.zeros(R)
    for i in range(nd - 1, 0, -1):
        if pr[i] > pr[i - 1]:
            pr[i - 1] = pr[i]
    idx = np.searchsorted(rc, rec_thrs, side="left")
    for ri, pi in enumerate(idx):
        if pi >= nd:
            break
        q[ri] = pr[pi]
        ss[ri] = sorted_scores[pi]
    return (rc[-1] if nd else 0), q, ss


def coco_evaluate(
    det_boxes: Sequence[np.ndarray],
    det_scores: Sequence[np.ndarray],
    det_labels: Sequence[np.ndarray],
    gt_boxes: Sequence[np.ndarray],
    gt_labels: Sequence[np.ndarray],
    gt_crowds: Optional[Sequence[np.ndarray]] = None,
    gt_areas: Optional[Sequence[np.ndarray]] = None,
    box_format: str = "xyxy",
    iou_thresholds: Optional[List[float]] = None,
    rec_thresholds: Optional[List[float]] = None,
    max_detection_thresholds: Optional[List[int]] = None,
    average: str = "macro",
    det_masks: Optional[Sequence[np.ndarray]] = None,
    gt_masks: Optional[Sequence[np.ndarray]] = None,
    iou_type: str = "bbox",
) -> Dict[str, np.ndarray]:
    """MeanAveragePrecision.compute for ONE IoU type (detection/mean_ap.py:521-598) with COCOeval restated inline.

    `det_masks` / `gt_masks` (per image bool [n, H, W]) = the metric was built with "segm" among its IoU types: a ground truth
    without a positive `area` then gets its MASK area (detection/mean_ap.py:920-925 — for the "bbox" evaluation of a
    ("bbox", "segm") metric as well), and `iou_type="segm"` evaluates mask IoUs (boxes may then be None).

    Inputs are per-image arrays (list position = image id, detection/mean_ap.py:886).  Returns the reference's result
    dict (numpy scalars/arrays) plus the raw `precision [T,R,K,A,M]`, `recall [T,K,A,M]`, `scores` tensors.
    """
    iou_thrs = np.array(iou_thresholds or default_iou_thresholds(), dtype=np.float64)
    rec_thrs = np.array(rec_thresholds or default_rec_thresholds(), dtype=np.float64)
    max_dets = sorted(max_detection_thresholds or [1, 10, 100])
    n_img = len(det_labels)
    if det_boxes is None:
        det_boxes = [np.zeros((len(np.asarray(x).reshape(-1)), 4), np.float32) for x in det_labels]
        gt_boxes = [np.zeros((len(np.asarray(x).reshape(-1)), 4), np.float32) for x in gt_labels]
    dboxes = [box_convert_to_xywh(np.asarray(b), box_format) for b in det_boxes]
    gboxes = [box_convert_to_xywh(np.asarray(b), box_format) for b in gt_boxes]
    segm = iou_type == "segm"
    if gt_masks is not None:
        det_masks = [np.asarray(m).astype(bool) for m in det_masks]
        gt_masks = [np.asarray(m).astype(bool) for m in gt_masks]
    dlab = [np.asarray(x).astype(np.int64).reshape(-1) for x in det_labels]
    glab = [np.asarray(x).astype(np.int64).reshape(-1) for x in gt_labels]
    dsc = [np.asarray(x).astype(np.float32).astype(np.float64).reshape(-1) for x in det_scores]
    gcr = [np.asarray(x).astype(np.int64).reshape(-1) if gt_crowds is not None else np.zeros(len(glab[i]), np.int64)
           for i, x in enumerate(gt_crowds if gt_crowds is not None else glab)]
    garea = []
    for i in range(n_img):
        wh = gboxes[i][:, 2].astype(np.float64) * gboxes[i][:, 3].astype(np.float64)
        if gt_masks is not None:
            wh = gt_masks[i].sum(axis=(1, 2)).astype(np.float64)
        if gt_areas is not None:
            given = np.asarray(gt_areas[i]).astype(np.float64).reshape(-1)
            wh = np.where(given > 0, given, wh)  # detection/mean_ap.py:920-925
        garea.append(wh)
    all_labels = np.concatenate(dlab + glab) if n_img else np.zeros(0, np.int64)
    classes = np.unique(all_labels)  # detection/mean_ap.py:861-865
    if average == "micro":  # :602-605 every label becomes class 0
        dlab = [np.zeros_like(x) for x in dlab]
        glab = [np.zeros_like(x) for x in glab]
        eval_classes = np.unique(np.concatenate(dlab + glab)) if n_img else np.zeros(0, np.int64)
    else:
        eval_classes = classes

    T, R, K, A, M = len(iou_thrs), len(rec_thrs), len(eval_classes), len(AREA_RANGES), len(max_dets)
    precision = -np.ones((T, R, K, A, M))
    recall = -np.ones((T, K, A, M))
    scores = -np.ones((T, R, K, A, M))
    stats = [-1.0] * 12
    if n_img > 0:
        # ---- evaluate (COCOeval.evaluate) ----
        evals = {}
        for k, cat in enumerate(eval_classes):
            for a, rng in enumerate(AREA_RANGES):
                for i in range(n_img):
                    dm, gm = dlab[i] == cat, glab[i] == cat
                    evals[k, a, i] = _evaluate_img((det_masks if segm else dboxes)[i][dm], dsc[i][dm],
                                                   (gt_masks if segm else gboxes)[i][gm], gcr[i][gm], garea[i][gm],
                                                   iou_thrs, rng, max_dets[-1], masks=segm)
        # ---- accumulate (COCOeval.accumulate) ----
        for k in range(K):
            for a in range(A):
                E = [evals[k, a, i] for i in range(n_img) if evals[k, a, i] is not None]
                if not E:
                    continue
                for m, max_det in enumerate(max_dets):
                    dt_scores = np.concatenate([e["scores"][:max_det] for e in E])
                    inds = np.argsort(-dt_scores, kind="mergesort")
                    sorted_scores = dt_scores[inds]
                    dtm = np.concatenate([e["dtm"][:, :max_det] for e in E], axis=1)[:, inds]
                    dt_ig = np.concatenate([e["dt_ig"][:, :max_det] for e in E], axis=1)[:, inds]
                    gt_ig = np.concatenate([e["gt_ig"] for e in E])
                    npig = np.count_nonzero(~gt_ig)
                    if npig == 0:
                        continue
                    tps = np.logical_and(dtm, np.logical_not(dt_ig))
                    fps = np.logical_and(np.logical_not(dtm), np.logical_not(dt_ig))
                    tp_sum = np.cumsum(tps, axis=1).astype(np.float64)
                    fp_sum = np.cumsum(fps, axis=1).astype(np.float64)
                    for t in range(T):
                        recall[t, k, a, m], precision[t, :, k, a, m], scores[t, :, k, a, m] = sample_pr_curve(
                            tp_sum[t], fp_sum[t], sorted_scores, npig, rec_thrs)

        # ---- summarize (COCOeval.summarize / _summarize) ----
        def summ(ap: bool, iou_thr=None, area=0, mdet=M - 1):
            s = precision if ap else recall
            if iou_thr is not None:
                sel = np.where(iou_thr == iou_thrs)[0]
                s = s[sel]
            s = s[:, :, :, area, mdet] if ap else s[:, :, area, mdet]
            vals = s[s > -1]
            return float(np.mean(vals)) if vals.size else -1.0

        stats = [summ(True), summ(True, 0.5), summ(True, 0.75), summ(True, area=1), summ(True, area=2), summ(True, area=3),
                 summ(False, mdet=0), summ(False, mdet=1), summ(False, mdet=2), summ(False, area=1), summ(False, area=2),
                 summ(False, area=3)]
    if n_img > 0 and (sum(len(x) for x in dlab) == 0 or sum(len(x) for x in glab) == 0):
        pass  # COCOeval still runs; with no gts of a class npig == 0 -> -1 everywhere, which `summ` reproduces
    names = ["map", "map_50", "map_75", "map_small", "map_medium", "map_large", f"mar_{max_dets[0]}", f"mar_{max_dets[1]}",
             f"mar_{max_dets[2]}", "mar_small", "mar_medium", "mar_large"]
    out = {n: np.float32(v) for n, v in zip(names, stats)}
    # per-class values (detection/mean_ap.py:562-588): categories are independent, so the per-class rerun of the
    # reference equals slicing the class axis of the macro evaluation
    if average == "macro" and K:
        mpc, rpc = [], []
        for k in range(K):
            s = precision[:, :, k, 0, M - 1]
            mpc.append(float(np.mean(s[s > -1])) if (s > -1).any() else -1.0)
            s = recall[:, k, 0, M - 1]
            rpc.append(float(np.mean(s[s > -1])) if (s > -1).any() else -1.0)
        out["map_per_class_values"] = np.array(mpc, dtype=np.float32)
        out[f"mar_{max_dets[-1]}_per_class_values"] = np.array(rpc, dtype=np.float32)
    out["classes"] = classes.astype(np.int32)
    out["precision"], out["recall"], out["scores"] = precision, recall, scores
    return out


# ---- the two phases of the device evaluation, as the records they exchange ----------------------------------------------
# The kernels (csrc/cocomap.cu) split COCOeval into a per-image MATCH phase that writes one record per detection and an
# ACCUMULATE phase that reads only those records (the sharded evaluation exchanges them between ranks).  These two functions
# restate COCOeval in that shape; `accumulate_records(*match_records(...))` is `coco_evaluate`'s precision / recall / scores.


def match_records(det_box, det_score, det_label, det_counts, gt_box, gt_label, gt_crowd, gt_area, gt_counts, classes,
                  iou_thresholds, max_det_last, micro=False, pair_inter=None, pair_off=None, det_mask_area=None,
                  gt_mask_area=None, gt_area_exact=False):
    """COCOeval.evaluateImg for every (image, class, area range) of the given images, written out per detection: class index
    (position of the label in the sorted `classes`; 0 for everything when `micro`), rank inside its (image, class) in
    COCOeval's order (`np.argsort(-score, kind="mergesort")`: descending, NaN last, +-0 equal, ties by input position), and
    uint64 match / ignore words with bit `area * T + threshold`; `npig` int32 [K, 4] counts the non-ignored ground truths.

    Flat inputs: xywh float32 boxes, float32 scores, int64 labels, per-image counts; `gt_area` is the given area (<= 0 or -0.0:
    w * h) unless `gt_area_exact`.  Mask mode (`pair_inter` not None): per image a flat [D, G] table of intersection pixel
    counts at `pair_off[image]`, IoU = maskApi.c:rleIou from it and the mask areas, a detection's area range from its mask
    area.  Only the first `max_det_last` detections of a (image, class) are matched; every detection gets a rank."""
    thr = np.asarray(iou_thresholds, np.float64)
    T = len(thr)
    cls = np.asarray(classes, np.int64).reshape(-1)
    K = 1 if micro else len(cls)
    det_counts, gt_counts = [int(x) for x in det_counts], [int(x) for x in gt_counts]
    n_det = sum(det_counts)
    cat = np.zeros(n_det, np.int32)
    rank = np.zeros(n_det, np.int32)
    match = np.zeros(n_det, np.uint64)
    ignore = np.zeros(n_det, np.uint64)
    npig = np.zeros((K, 4), np.int32)
    dbox = np.asarray(det_box, np.float32).reshape(-1, 4)
    gbox = np.asarray(gt_box, np.float32).reshape(-1, 4)
    dscore = np.asarray(det_score, np.float32).reshape(-1)
    dlab, glab = np.asarray(det_label, np.int64).reshape(-1), np.asarray(gt_label, np.int64).reshape(-1)
    gcrowd = np.asarray(gt_crowd).reshape(-1) != 0
    given = np.asarray(gt_area, np.float64).reshape(-1)
    gt_wh = gbox[:, 2].astype(np.float64) * gbox[:, 3].astype(np.float64)
    garea = given if gt_area_exact else np.where(given > 0, given, gt_wh)
    masks = pair_inter is not None
    d0 = g0 = 0
    for img, (nd, ng) in enumerate(zip(det_counts, gt_counts)):
        dcat = np.zeros(nd, np.int64) if micro else np.searchsorted(cls, dlab[d0:d0 + nd])
        gcat = np.zeros(ng, np.int64) if micro else np.searchsorted(cls, glab[g0:g0 + ng])
        cat[d0:d0 + nd] = dcat
        if masks:
            table = np.asarray(pair_inter, np.float64)[int(pair_off[img]): int(pair_off[img]) + nd * ng].reshape(nd, ng)
        for c in np.unique(np.concatenate([dcat, gcat])):
            di, gi = np.flatnonzero(dcat == c), np.flatnonzero(gcat == c)
            order = di[np.argsort(-dscore[d0 + di], kind="mergesort")]
            rank[d0 + order] = np.arange(len(order))
            top = order[:max_det_last]
            for a, (lo, hi) in enumerate(AREA_RANGES):
                g_ig = gcrowd[g0 + gi] | (garea[g0 + gi] < lo) | (garea[g0 + gi] > hi)
                npig[c, a] += int((~g_ig).sum())
                g_order = gi[np.argsort(g_ig, kind="mergesort")]
                crowd_sorted = gcrowd[g0 + g_order]
                if masks:
                    inter = table[np.ix_(top, g_order)]
                    da = np.asarray(det_mask_area, np.float64)[d0 + top][:, None]
                    ga = np.asarray(gt_mask_area, np.float64)[g0 + g_order][None, :]
                    with np.errstate(divide="ignore", invalid="ignore"):
                        ious = np.where(inter > 0, inter / np.where(crowd_sorted[None, :], da, da + ga - inter), 0.0)
                    d_area = np.asarray(det_mask_area, np.float64)[d0 + top]
                else:
                    ious = bb_iou(dbox[d0 + top], gbox[g0 + g_order], crowd_sorted)
                    d_area = dbox[d0 + top, 2].astype(np.float64) * dbox[d0 + top, 3].astype(np.float64)
                dtm, dt_ig = match_detections(ious, crowd_sorted, g_ig[np.argsort(g_ig, kind="mergesort")], thr)
                dt_ig = dt_ig | ((dtm == 0) & ((d_area < lo) | (d_area > hi))[None, :])
                for t in range(T):
                    bit = np.uint64(1) << np.uint64(a * T + t)
                    match[d0 + top[dtm[t] > 0]] |= bit
                    ignore[d0 + top[dt_ig[t]]] |= bit
        d0, g0 = d0 + nd, g0 + ng
    return cat, rank, match, ignore, npig


def accumulate_records(det_cat, det_score, det_rank, det_match, det_ignore, npig, num_classes, class_lo, class_hi, n_iou_thr,
                       rec_thresholds, max_dets):
    """COCOeval.accumulate from the per-detection records for the classes [class_lo, class_hi): per (class, area, maxDet) the
    records of the class with rank < maxDet in COCOeval's score order (ties keep the order the records are given in), TP / FP
    running sums, `sample_pr_curve`.  Full-size float64 `precision [T,R,K,4,M]`, `recall [T,K,4,M]`, `scores`, -1 outside the
    range and where `npig == 0`."""
    T, R, K, M = int(n_iou_thr), len(rec_thresholds), int(num_classes), len(max_dets)
    rec = np.asarray(rec_thresholds, np.float64)
    precision, recall, scores = -np.ones((T, R, K, 4, M)), -np.ones((T, K, 4, M)), -np.ones((T, R, K, 4, M))
    cat, rank = np.asarray(det_cat).reshape(-1), np.asarray(det_rank).reshape(-1)
    score = np.asarray(det_score, np.float32).reshape(-1).astype(np.float64)
    match = np.asarray(det_match).reshape(-1).view(np.uint64)
    ignore = np.asarray(det_ignore).reshape(-1).view(np.uint64)
    n_valid = np.asarray(npig).reshape(-1, 4)
    by_class = np.argsort(cat, kind="stable")
    start = np.searchsorted(cat[by_class], np.arange(K + 1))
    for k in range(int(class_lo), int(class_hi)):
        in_class = by_class[start[k]:start[k + 1]]  # input order
        for a in range(4):
            if n_valid[k, a] == 0:
                continue
            for m, max_det in enumerate(max_dets):
                sel = in_class[rank[in_class] < max_det]
                sel = sel[np.argsort(-score[sel], kind="mergesort")]
                for t in range(T):
                    bit = np.uint64(1) << np.uint64(a * T + t)
                    hit, ign = (match[sel] & bit) != 0, (ignore[sel] & bit) != 0
                    tp = np.cumsum(hit & ~ign).astype(np.float64)
                    fp = np.cumsum(~hit & ~ign).astype(np.float64)
                    recall[t, k, a, m], precision[t, :, k, a, m], scores[t, :, k, a, m] = sample_pr_curve(
                        tp, fp, score[sel], n_valid[k, a], rec)
    return precision, recall, scores
