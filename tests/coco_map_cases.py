"""Hand-built COCO mAP cases (flat, xywh) at the edges of the matching and accumulation rules, shared by the record-level
oracle check on the CPU (tests/test_oracle_map.py) and the kernel path suite (tests/test_coco_map_paths_gpu.py).

A case is a dict of flat arrays: `det_box` / `gt_box` float32 [n, 4] xywh, `det_score` float32, `det_label` / `gt_label`
int64, `gt_crowd` uint8, `gt_area` float64 (the given area; <= 0 falls back to w * h), per-image `det_counts` / `gt_counts`,
`iou_thr`, `rec_thr`, three `max_dets`, `micro`; mask cases add per-image boolean `det_masks` / `gt_masks` [n, H, W]."""
import numpy as np

from oracle.coco_map import coco_evaluate, default_iou_thresholds, default_rec_thresholds, match_records

NAN, INF = float("nan"), float("inf")


def make_case(images, iou_thr=None, max_dets=(1, 10, 100), micro=False, rec_thr=None):
    """`images`: per image a dict with `det` [(x, y, w, h, score, label)], `gt` [(x, y, w, h, label, crowd, area)] and
    optionally `det_masks` / `gt_masks`."""
    det = [d for im in images for d in im.get("det", [])]
    gt = [g for im in images for g in im.get("gt", [])]
    case = dict(
        det_box=np.array([d[:4] for d in det], np.float32).reshape(-1, 4),
        det_score=np.array([d[4] for d in det], np.float32),
        det_label=np.array([d[5] for d in det], np.int64),
        det_counts=[len(im.get("det", [])) for im in images],
        gt_box=np.array([g[:4] for g in gt], np.float32).reshape(-1, 4),
        gt_label=np.array([g[4] for g in gt], np.int64),
        gt_crowd=np.array([g[5] for g in gt], np.uint8),
        gt_area=np.array([g[6] for g in gt], np.float64),
        gt_counts=[len(im.get("gt", [])) for im in images],
        iou_thr=list(iou_thr or default_iou_thresholds()),
        rec_thr=list(rec_thr or default_rec_thresholds()),
        max_dets=list(max_dets),
        micro=micro,
    )
    if any("det_masks" in im for im in images):
        case["det_masks"] = [np.asarray(im["det_masks"], bool) for im in images]
        case["gt_masks"] = [np.asarray(im["gt_masks"], bool) for im in images]
    return case


def classes_of(case):
    return np.unique(np.concatenate([case["det_label"], case["gt_label"]]))


def mask_inputs(case):
    """Mask mode: the per-image [D, G] intersection tables (exact integer pixel counts), their offsets, both mask areas and
    the ground-truth areas resolved like detection/mean_ap.py:920-925 (given if > 0, else the mask area)."""
    inter, off, pos = [], [], 0
    for dm, gm in zip(case["det_masks"], case["gt_masks"]):
        d = dm.reshape(len(dm), -1).astype(np.int64)
        g = gm.reshape(len(gm), -1).astype(np.int64)
        t = (d @ g.T).astype(np.float64).reshape(-1)
        off.append(pos)
        inter.append(t)
        pos += t.size
    det_area = np.concatenate([m.reshape(len(m), -1).sum(1) for m in case["det_masks"]]).astype(np.float64)
    gt_area = np.concatenate([m.reshape(len(m), -1).sum(1) for m in case["gt_masks"]]).astype(np.float64)
    if not case["micro"]:  # the pair kernel writes 0 for a pair of different classes; the matcher never reads it
        d0 = g0 = 0
        for i, (nd, ng) in enumerate(zip(case["det_counts"], case["gt_counts"])):
            same = case["det_label"][d0:d0 + nd, None] == case["gt_label"][None, g0:g0 + ng]
            inter[i] = inter[i] * same.reshape(-1)
            d0, g0 = d0 + nd, g0 + ng
    resolved = np.where(case["gt_area"] > 0, case["gt_area"], gt_area)
    return dict(pair_inter=np.concatenate(inter + [np.zeros(0)]), pair_off=np.array(off, np.int64), det_mask_area=det_area,
                gt_mask_area=gt_area, gt_area=resolved)


def oracle_records(case):
    kw = {}
    gt_area = case["gt_area"]
    if "det_masks" in case:
        m = mask_inputs(case)
        gt_area = m.pop("gt_area")
        kw = dict(m, gt_area_exact=True)
    return match_records(case["det_box"], case["det_score"], case["det_label"], case["det_counts"], case["gt_box"],
                         case["gt_label"], case["gt_crowd"], gt_area, case["gt_counts"], classes_of(case), case["iou_thr"],
                         case["max_dets"][-1], micro=case["micro"], **kw)


def coco_eval(case):
    """`coco_evaluate` (COCOeval restated per image) on the case."""
    def split(x, counts):
        return np.split(np.asarray(x), np.cumsum(counts)[:-1]) if len(counts) else []

    dc, gc = case["det_counts"], case["gt_counts"]
    segm = "det_masks" in case
    return coco_evaluate(
        None if segm else split(case["det_box"], dc), split(case["det_score"], dc), split(case["det_label"], dc),
        None if segm else split(case["gt_box"], gc), split(case["gt_label"], gc), split(case["gt_crowd"], gc),
        split(case["gt_area"], gc), box_format="xywh", iou_thresholds=case["iou_thr"], rec_thresholds=case["rec_thr"],
        max_detection_thresholds=case["max_dets"], average="micro" if case["micro"] else "macro",
        det_masks=case.get("det_masks"), gt_masks=case.get("gt_masks"), iou_type="segm" if segm else "bbox")


# ---- the cases ----------------------------------------------------------------------------------------------------------
F055 = 9227469  # float32(0.55) == 9227469 / 2**24 exactly: torch.linspace(0.5, 0.95, 10)[1]


def iou_at_threshold():
    """IoU exactly equal to a threshold matches (`iou < best` skips only smaller ones); one float32 ulp below does not."""
    big = float(2 ** 24)
    return make_case([
        dict(det=[(0, 0, big, 1, 0.9, 1)], gt=[(0, 0, F055, 1, 1, 0, 0)]),          # IoU == float32(0.55)
        dict(det=[(0, 0, big, 1, 0.9, 1)], gt=[(0, 0, F055 - 1, 1, 1, 0, 0)]),      # one ulp below
        dict(det=[(0, 0, 2, 1, 0.8, 1)], gt=[(0, 0, 1, 1, 1, 0, 0)]),               # 0.5
        dict(det=[(0, 0, 4, 1, 0.7, 1)], gt=[(0, 0, 3, 1, 1, 0, 0)]),               # 0.75
        dict(det=[(1, 0, 3, 1, 0.6, 1)], gt=[(0, 0, 4, 1, 1, 0, 0)]),               # 0.75, offset box
    ])


def equal_iou_ties():
    """Two ground truths at the same IoU: the later one wins, among non-ignored and among ignored (crowd) ones; a
    non-ignored match is kept even when an ignored ground truth overlaps more."""
    return make_case([
        dict(det=[(0, 0, 10, 10, 0.9, 0)], gt=[(0, 0, 10, 5, 0, 0, 0), (0, 5, 10, 5, 0, 0, 0)]),
        dict(det=[(0, 0, 10, 10, 0.9, 0), (0, 0, 10, 10, 0.8, 0)],
             gt=[(0, 0, 10, 5, 0, 1, 0), (0, 5, 10, 5, 0, 1, 0)]),
        dict(det=[(0, 0, 10, 10, 0.9, 0)], gt=[(0, 0, 10, 6, 0, 0, 0), (0, 0, 10, 10, 0, 1, 0)]),
        dict(det=[(0, 0, 10, 10, 0.9, 0), (0, 0, 10, 10, 0.5, 0)],
             gt=[(0, 0, 10, 10, 0, 0, 5000.0), (0, 0, 10, 10, 0, 0, 50.0)]),  # equal IoU, the small-area one ignored in "medium"
    ], iou_thr=[0.3, 0.5, 0.6, 0.99])


def crowd_reuse():
    """A crowd ground truth is matched by every detection inside it (union = the detection's area)."""
    return make_case([
        dict(det=[(10, 10, 20, 20, s, 3) for s in (0.9, 0.8, 0.7)] + [(0, 0, 100, 100, 0.6, 3), (5, 5, 50, 50, 0.5, 3)],
             gt=[(0, 0, 100, 100, 3, 1, 0), (10, 10, 20, 20, 3, 0, 0)]),
    ], iou_thr=[0.1, 0.5, 0.95])


def area_bounds():
    """Areas 1024 and 9216 lie in both neighbouring ranges (inclusive bounds); 1023.9999 / 1024.0001 on one side; a given
    area <= 0, -0.0 or negative falls back to w * h; unmatched detections of area 1024 / 9216 are ignored by range."""
    gts = [(0, 0, 10, 10, 0, 0, a) for a in (1024.0, 9216.0, 1023.9999, 1024.0001, 9215.9999, 9216.0001)]
    gts += [(200, 0, 32, 32, 0, 0, 0.0), (300, 0, 96, 96, 0, 0, -0.0), (400, 0, 32, 32, 0, 0, -5.0),
            (600, 0, 96, 96, 0, 0, 0.0)]
    dets = [(0, 0, 10, 10, 0.9 - 0.01 * i, 0) for i in range(6)]
    dets += [(200, 0, 32, 32, 0.5, 0), (300, 0, 96, 96, 0.4, 0), (400, 0, 32, 32, 0.3, 0)]
    dets += [(1000, 1000, 32, 32, 0.2, 0), (2000, 2000, 96, 96, 0.1, 0), (3000, 0, 32.0, 31.999, 0.05, 0)]
    return make_case([dict(det=dets, gt=gts)], iou_thr=[0.5, 0.9])


def degenerate_boxes():
    """Zero-width, negative-width and empty boxes on both sides (IoU 0, area w * h <= 0)."""
    return make_case([
        dict(det=[(0, 0, 0, 10, 0.9, 1), (0, 0, -3, 10, 0.8, 1), (0, 0, 0, 0, 0.7, 1), (0, 0, 10, 10, 0.6, 1)],
             gt=[(0, 0, 0, 10, 1, 0, 0), (0, 0, -3, 10, 1, 0, 0), (0, 0, 0, 0, 1, 0, 0), (0, 0, 10, 10, 1, 0, 0)]),
        dict(det=[(5, 5, 0, 0, 0.5, 1)], gt=[(5, 5, 0, 0, 1, 1, 0)]),
    ], iou_thr=[0.0, 0.5])


def _label_images(labels):
    rng = np.random.default_rng(11)
    images = []
    for _ in range(3):
        det, gt = [], []
        for lab in labels:
            for _ in range(int(rng.integers(0, 3))):
                x, y = (int(v) for v in rng.integers(0, 40, 2))
                gt.append((x, y, 20, 20, lab, 0, 0))
                det.append((x + int(rng.integers(0, 6)), y, 20, 20, float(rng.integers(1, 8)) / 8, lab))
            if rng.random() < 0.5:
                det.append((100, 100, 10, 10, 0.3, lab))
        images.append(dict(det=det, gt=gt))
    return images


def label_values():
    """Large, negative and gapped labels go through the sorted class list (`class_index`)."""
    return make_case(_label_images([-7, 0, 3, 1 << 40, -(1 << 33), 12]))


def label_values_micro():
    return make_case(_label_images([-7, 0, 3, 1 << 40, -(1 << 33), 12]), micro=True)


def tied_scores():
    """All-equal scores within and across images; ties straddling the max_det cut (ranks break ties by index)."""
    rng = np.random.default_rng(3)
    images = []
    for i in range(3):
        det = [(int(rng.integers(0, 30)), int(rng.integers(0, 30)), 20, 20, 0.5, 0) for _ in range(12)]
        det += [(int(rng.integers(0, 30)), 0, 20, 20, 0.25 if j % 2 else 0.75, 1) for j in range(9)]
        gt = [(int(rng.integers(0, 30)), int(rng.integers(0, 30)), 20, 20, c, 0, 0) for c in (0, 0, 0, 1, 1)]
        images.append(dict(det=det, gt=gt))
    return make_case(images, max_dets=(1, 4, 7))


def nan_scores():
    """NaN scores: COCOeval's mergesort puts them after every other score, -inf included, in input order."""
    return make_case([
        dict(det=[(0, 0, 10, 10, 0.3, 0), (0, 0, 10, 10, NAN, 0), (0, 0, 10, 10, 0.9, 0), (0, 0, 10, 10, 0.9, 0)],
             gt=[(0, 0, 10, 10, 0, 0, 0), (1, 0, 10, 10, 0, 0, 0)]),
        dict(det=[(0, 0, 10, 10, NAN, 0), (0, 0, 10, 10, -INF, 0), (0, 0, 10, 10, NAN, 0), (0, 0, 10, 10, 0.1, 0),
                  (0, 0, 10, 10, NAN, 1)],
             gt=[(0, 0, 10, 10, 0, 0, 0), (0, 0, 10, 10, 1, 0, 0)]),
    ], max_dets=(1, 2, 3))


def signed_zero_inf_scores():
    """+-0 tie (kept in input order), +-inf order at the ends."""
    return make_case([
        dict(det=[(0, 0, 10, 10, -0.0, 0), (0, 0, 10, 10, 0.0, 0), (0, 0, 10, 10, INF, 0), (0, 0, 10, 10, -INF, 0),
                  (0, 0, 10, 10, -0.0, 0), (2, 0, 10, 10, 0.0, 0)],
             gt=[(0, 0, 10, 10, 0, 0, 0), (2, 0, 10, 10, 0, 0, 0), (0, 1, 10, 10, 0, 0, 0)]),
        dict(det=[(0, 0, 10, 10, 0.0, 0), (0, 0, 10, 10, -0.0, 0)], gt=[(0, 0, 10, 10, 0, 0, 0)]),
    ], max_dets=(1, 2, 4))


def _masks(rng, n, h, w, p):
    return rng.random((n, h, w)) < p


def mask_edges():
    """Mask mode: an empty detection mask and an empty ground-truth mask (intersection 0 -> IoU 0), a crowd ground truth
    (union = the detection's mask area), given areas next to mask areas, a detection's area range from its mask area."""
    rng = np.random.default_rng(5)
    h, w = 6, 7
    dm = _masks(rng, 5, h, w, 0.6)
    dm[1] = False
    gm = _masks(rng, 4, h, w, 0.6)
    gm[2] = False
    gm[3] = True
    im0 = dict(det=[(0, 0, 1, 1, s, lab) for s, lab in zip((0.9, 0.8, 0.7, 0.6, 0.5), (0, 0, 0, 1, 1))],
               gt=[(0, 0, 1, 1, 0, 0, 0), (0, 0, 1, 1, 0, 0, 2000.0), (0, 0, 1, 1, 0, 0, 0), (0, 0, 1, 1, 1, 1, 0)],
               det_masks=dm, gt_masks=gm)
    big = np.zeros((2, 40, 40), bool)
    big[0, :33, :32] = True  # 1056 pixels: "medium"
    big[1, :32, :32] = True  # 1024: "small" and "medium"
    im1 = dict(det=[(0, 0, 1, 1, 0.4, 0), (0, 0, 1, 1, 0.4, 0)], gt=[(0, 0, 1, 1, 0, 0, 0)], det_masks=big,
               gt_masks=big[1:])
    return make_case([im0, im1], iou_thr=[0.1, 0.5, 0.75])


def mask_edges_micro():
    c = mask_edges()
    c["micro"] = True
    return c


HAND_BUILT = {f.__name__: f for f in (iou_at_threshold, equal_iou_ties, crowd_reuse, area_bounds, degenerate_boxes,
                                      label_values, label_values_micro, tied_scores, nan_scores, signed_zero_inf_scores,
                                      mask_edges, mask_edges_micro)}
