"""COCO-style mean average precision / recall for object detection (reference: detection/mean_ap.py).

The reference stores per-image tensors, then at ``compute`` copies every number to host Python objects and lets
``pycocotools`` do all the arithmetic on the CPU.  Here the nine list states and their per-image layout are kept (same
names, ``dist_reduce_fx=None``), but ``compute`` concatenates them once on the device and runs three kernels
(`mb200_coco_map_evaluate`, csrc/cocomap.cu): per-image matching, a stable radix sort by (class, score), per-(class,
area, maxDet) accumulation.

``iou_type="segm"`` (reference :848-853, :897-944): the reference run-length encodes every mask on the host at ``update`` and
pycocotools intersects the codes pair by pair on the host at ``compute``.  Here ``update`` packs the masks to one bit per pixel
on the device (`mb200_mask_pack_bits`; the state entry of an image is ONE int32 tensor ``[n, H, W, areas.., bit words..]``),
``compute`` builds every image's [detections x ground truths] table of intersection pixel counts with one launch
(`mb200_mask_pair_intersections`) and the matching kernel reads IoUs from it (`mb200_coco_map_match_ex`).  COCO json of masks
(``coco_to_tm`` / ``tm_to_coco`` with segm): run-length codes, host side (detection/rle.py); polygons are not supported.
"""
from __future__ import annotations

import os

import json
from typing import Any, Dict, List, Optional, Tuple, Union

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200 import _native
from metrics_b200.detection.helpers import _fix_empty_tensors, _input_validator
from metrics_b200.metric import Metric
from metrics_b200.utilities.prints import rank_zero_warn


def _box_convert_to_xywh(boxes: Tensor, in_fmt: str) -> Tensor:
    """torchvision.ops.box_convert(boxes, in_fmt, "xywh") restated op for op (fp32 rounding matters for parity):
    cxcywh goes through xyxy first (reference detection/mean_ap.py:846)."""
    if in_fmt == "xywh":
        return boxes
    if in_fmt == "cxcywh":
        cx, cy, w, h = boxes.unbind(-1)
        boxes = torch.stack((cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h), dim=-1)
    x1, y1, x2, y2 = boxes.unbind(-1)
    return torch.stack((x1, y1, x2 - x1, y2 - y1), dim=-1)


def _pairwise_ious(det_box: Tensor, det_score: Tensor, det_label: Tensor, det_counts: List[int], gt_box: Tensor,
                   gt_label: Tensor, gt_crowd: Tensor, gt_counts: List[int], classes: List[int], micro: bool,
                   max_det: int, masks: Optional[Dict[str, Tensor]] = None) -> Dict[Tuple[int, int], Any]:
    """The ``ious`` entry of the extended summary (reference :552-555, i.e. pycocotools ``COCOeval.computeIoU`` for every
    (image, category)): ``{(image, class): [D, G] float32}`` with the pair's detections in descending-score order (stable,
    cut to the largest max-detection threshold) and its ground truths in input order; ``[]`` when either side is empty.

    pycocotools fills the dict with one small host computation per (image, category).  Here ALL pairs of the whole state
    are evaluated by one batch of device ops over a flat pair list (fp64, crowd ground truths use the detection's area as
    the union, ``maskApi.c:bbIou``); the dict values are views into that one tensor."""
    dev = det_box.device
    n_img, n_cls = len(det_counts), (1 if micro else len(classes))
    img_of_det = torch.repeat_interleave(torch.arange(n_img, device=dev), torch.tensor(det_counts, device=dev))
    img_of_gt = torch.repeat_interleave(torch.arange(n_img, device=dev), torch.tensor(gt_counts, device=dev))
    if micro:
        det_key, gt_key = img_of_det, img_of_gt
    else:
        table = torch.tensor(classes, dtype=torch.int64, device=dev)
        det_key = img_of_det * n_cls + torch.searchsorted(table, det_label)
        gt_key = img_of_gt * n_cls + torch.searchsorted(table, gt_label)
    # detections: by (pair, score descending, input order) in COCOeval's order (`argsort(-score, kind="mergesort")`): an
    # ascending sort of `0 - score` puts NaN last and turns -0.0 into +0.0, so that +-0 tie; ground truths: by (pair, input order)
    by_score = torch.sort(0.0 - det_score, stable=True).indices
    det_order = by_score[torch.sort(det_key[by_score], stable=True).indices]
    gt_order = torch.sort(gt_key, stable=True).indices
    n_pairs = n_img * n_cls
    det_total = torch.bincount(det_key, minlength=n_pairs)
    gt_cnt = torch.bincount(gt_key, minlength=n_pairs)
    det_start = torch.cumsum(det_total, 0) - det_total
    gt_start = torch.cumsum(gt_cnt, 0) - gt_cnt
    sorted_key = det_key[det_order]
    rank = torch.arange(det_order.numel(), device=dev) - det_start[sorted_key]
    keep = rank < max_det
    det_order, sorted_key = det_order[keep], sorted_key[keep]
    det_cnt = torch.clamp(det_total, max=max_det)
    # flat list of (detection row, ground-truth column) pairs, row-major inside every (image, class) block
    cols_of_row = gt_cnt[sorted_key]
    row = torch.repeat_interleave(torch.arange(det_order.numel(), device=dev), cols_of_row)
    row_first = torch.cumsum(cols_of_row, 0) - cols_of_row
    col = torch.arange(row.numel(), device=dev) - row_first[row]
    d_index = det_order[row]
    g_index = gt_order[gt_start[sorted_key[row]] + col]
    if masks is None:
        d = det_box[d_index].to(torch.float64)
        g = gt_box[g_index].to(torch.float64)
        w = torch.minimum(d[:, 0] + d[:, 2], g[:, 0] + g[:, 2]) - torch.maximum(d[:, 0], g[:, 0])
        h = torch.minimum(d[:, 1] + d[:, 3], g[:, 1] + g[:, 3]) - torch.maximum(d[:, 1], g[:, 1])
        inter = torch.where((w > 0) & (h > 0), w * h, torch.zeros_like(w))
        det_area = d[:, 2] * d[:, 3]
        union = torch.where(gt_crowd[g_index] != 0, det_area, det_area + g[:, 2] * g[:, 3] - inter)
        flat = (inter / union).to(torch.float32)
    else:  # instance masks: the per-image [D, G] tables of intersection pixel counts (maskApi.c:rleIou semantics)
        det_counts_t, gt_counts_t = torch.tensor(det_counts, device=dev), torch.tensor(gt_counts, device=dev)
        det_first = torch.cumsum(det_counts_t, 0) - det_counts_t
        gt_first = torch.cumsum(gt_counts_t, 0) - gt_counts_t
        img = img_of_det[d_index]
        inter = masks["pair_inter"][masks["pair_off"][img] + (d_index - det_first[img]) * gt_counts_t[img] + (g_index - gt_first[img])]
        det_area = masks["det_area"][d_index]
        union = torch.where(gt_crowd[g_index] != 0, det_area, det_area + masks["gt_area"][g_index] - inter)
        flat = torch.where(inter > 0, inter / union, torch.zeros_like(inter)).to(torch.float32)
    # one host read of the block shapes, then the dict is assembled from views
    shapes = torch.stack((det_cnt, gt_cnt), 1).cpu().tolist()
    out: Dict[Tuple[int, int], Any] = {}
    offset = 0
    for pair, (n_d, n_g) in enumerate(shapes):
        key = (pair // n_cls, 0 if micro else classes[pair % n_cls])
        if n_d == 0 or n_g == 0:
            out[key] = []
            continue
        out[key] = flat[offset: offset + n_d * n_g].view(n_d, n_g)
        offset += n_d * n_g
    return out


class MeanAveragePrecision(Metric):
    """mAP / mAR for object detection and instance segmentation (reference :77-1063).

    ``update(preds, target)``: lists (one entry per image) of dicts with ``boxes [n,4]`` (``iou_type`` bbox) and / or ``masks
    [n,H,W]`` bool (segm), ``scores [n]``, ``labels [n]`` (preds) and the same geometry keys, ``labels`` and optional
    ``iscrowd``, ``area`` (target).  With both IoU types the result keys carry a ``bbox_`` / ``segm_`` prefix.  ``compute()`` returns the
    reference's dict: ``map, map_50, map_75, map_small/medium/large, mar_{d1,d2,d3}, mar_small/medium/large,
    map_per_class, mar_{d3}_per_class, classes`` (+ ``precision / recall / scores`` with ``extended_summary``).
    """

    is_differentiable: bool = False
    higher_is_better: Optional[bool] = True
    full_state_update: bool = True
    plot_lower_bound: float = 0.0
    plot_upper_bound: float = 1.0

    warn_on_many_detections: bool = True

    def __init__(
        self,
        box_format: Literal["xyxy", "xywh", "cxcywh"] = "xyxy",
        iou_type: Union[Literal["bbox", "segm"], Tuple[str]] = "bbox",
        iou_thresholds: Optional[List[float]] = None,
        rec_thresholds: Optional[List[float]] = None,
        max_detection_thresholds: Optional[List[int]] = None,
        class_metrics: bool = False,
        extended_summary: bool = False,
        average: Literal["macro", "micro"] = "macro",
        backend: Literal["pycocotools", "faster_coco_eval"] = "pycocotools",
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        allowed_box_formats = ("xyxy", "xywh", "cxcywh")
        if box_format not in allowed_box_formats:
            raise ValueError(f"Expected argument `box_format` to be one of {allowed_box_formats} but got {box_format}")
        self.box_format = box_format
        if isinstance(iou_type, str):
            iou_type = (iou_type,)
        if any(tp not in ("bbox", "segm") for tp in iou_type):
            raise ValueError(f"Expected argument `iou_type` to be one of ('bbox', 'segm') or a tuple of, but got {iou_type}")
        self.iou_type = tuple(iou_type)

        if iou_thresholds is not None and not isinstance(iou_thresholds, list):
            raise ValueError(
                f"Expected argument `iou_thresholds` to either be `None` or a list of floats but got {iou_thresholds}"
            )
        self.iou_thresholds = iou_thresholds or torch.linspace(0.5, 0.95, round((0.95 - 0.5) / 0.05) + 1).tolist()
        if rec_thresholds is not None and not isinstance(rec_thresholds, list):
            raise ValueError(
                f"Expected argument `rec_thresholds` to either be `None` or a list of floats but got {rec_thresholds}"
            )
        self.rec_thresholds = rec_thresholds or torch.linspace(0.0, 1.00, round(1.00 / 0.01) + 1).tolist()
        if max_detection_thresholds is not None and not isinstance(max_detection_thresholds, list):
            raise ValueError(
                f"Expected argument `max_detection_thresholds` to either be `None` or a list of ints"
                f" but got {max_detection_thresholds}"
            )
        if max_detection_thresholds is not None and len(max_detection_thresholds) != 3:
            raise ValueError(
                "When providing a list of max detection thresholds it should have length 3."
                f" Got value {len(max_detection_thresholds)}"
            )
        self.max_detection_thresholds = sorted(int(x) for x in (max_detection_thresholds or [1, 10, 100]))
        if not isinstance(class_metrics, bool):
            raise ValueError("Expected argument `class_metrics` to be a boolean")
        self.class_metrics = class_metrics
        if not isinstance(extended_summary, bool):
            raise ValueError("Expected argument `extended_summary` to be a boolean")
        self.extended_summary = extended_summary
        if average not in ("macro", "micro"):
            raise ValueError(f"Expected argument `average` to be one of ('macro', 'micro') but got {average}")
        self.average = average
        if backend not in ("pycocotools", "faster_coco_eval"):
            raise ValueError(
                f"Expected argument `backend` to be one of ('pycocotools', 'faster_coco_eval') but got {backend}"
            )
        self.backend = backend  # accepted for API compatibility; the evaluation always runs on the device

        for name in ("detection_box", "detection_mask", "detection_scores", "detection_labels", "groundtruth_box",
                     "groundtruth_mask", "groundtruth_labels", "groundtruth_crowds", "groundtruth_area"):
            self.add_state(name, default=[], dist_reduce_fx=None)

    # ------------------------------------------------------------------------------------------------
    def update(self, preds: List[Dict[str, Tensor]], target: List[Dict[str, Tensor]]) -> None:
        """Append one entry per image to the list states (reference :478-519).  Box conversion to xywh runs as ONE
        batched op per call; the per-image states are views into it."""
        _input_validator(preds, target, iou_type=self.iou_type)
        limit = self.max_detection_thresholds[-1]
        if self.warn_on_many_detections and any(len(p["labels"]) > limit for p in preds):
            rank_zero_warn(
                f"Encountered more than {limit} detections in a single image. This means that certain detections with "
                "the lowest scores will be ignored, that may have an undesirable impact on performance. Please consider"
                " adjusting the `max_detection_threshold` to suit your use case. To disable this warning, set attribute "
                "class `warn_on_many_detections=False`, after initializing the metric.",
                UserWarning,
            )
        if "segm" in self.iou_type:  # reference :848-853 (host RLE per mask); here: bit-packed on the device, one entry per image
            self.detection_mask.extend(self._mask_state(p["masks"]) for p in preds)
            self.groundtruth_mask.extend(self._mask_state(t["masks"]) for t in target)
        box_sources = () if "bbox" not in self.iou_type else (
            ([_fix_empty_tensors(p["boxes"]) for p in preds], self.detection_box),
            ([_fix_empty_tensors(t["boxes"]) for t in target], self.groundtruth_box))
        for boxes_list, store in box_sources:
            counts = [b.shape[0] if b.numel() > 0 else 0 for b in boxes_list]
            nonempty = [b if b.ndim == 2 else b.reshape(-1, 4) for b in boxes_list if b.numel() > 0]
            if nonempty:
                converted = _box_convert_to_xywh(torch.cat(nonempty), self.box_format)
                pieces = iter(converted.split([c for c in counts if c > 0]))
            for b, c in zip(boxes_list, counts):
                store.append(next(pieces) if c > 0 else b)
        self.detection_labels.extend([item["labels"] for item in preds])
        self.detection_scores.extend([item["scores"] for item in preds])
        # defaults for missing `iscrowd` / `area` (reference :518: zeros_like(labels) per image): ONE zero buffer per call,
        # handed out as per-image views — a launch per image would dominate the whole update otherwise
        zero_views = None
        if target and any("iscrowd" not in t or "area" not in t for t in target):
            first = target[0]["labels"]
            zero_views = torch.zeros(sum(int(t["labels"].shape[0]) for t in target), dtype=first.dtype,
                                     device=first.device).split([int(t["labels"].shape[0]) for t in target])
        for i, item in enumerate(target):
            labels = item["labels"]
            self.groundtruth_labels.append(labels)
            default = None
            if zero_views is not None:
                default = zero_views[i] if (labels.dtype == zero_views[i].dtype and labels.ndim == 1) else torch.zeros_like(labels)
            self.groundtruth_crowds.append(item["iscrowd"] if "iscrowd" in item else default)
            self.groundtruth_area.append(item["area"] if "area" in item else default)

    # ------------------------------------------------------------------------------------------------
    # instance masks (iou_type "segm")
    # ------------------------------------------------------------------------------------------------
    def _mask_state(self, masks: Tensor) -> Tensor:
        """``[n, H, W]`` boolean masks -> the image's state entry: int32 ``[n, H, W, area_0..area_{n-1}, bit words (n rows of
        ceil(H*W/32), pixel order)]`` on the metric's device (`mb200_mask_pack_entry`)."""
        if masks.ndim != 3:
            if masks.numel() != 0:
                raise ValueError(f"Expected `masks` of shape (num_masks, height, width) but got {tuple(masks.shape)}")
            masks = masks.reshape(0, 0, 0)  # e.g. `coco_to_tm` of an image without detections
        return _native.mask_pack_entry(masks.to(self.device))  # one memset + one launch, no host -> device copy

    def _mask_tables(self, det_label: Tensor, gt_label: Tensor, det_counts: List[int], gt_counts: List[int],
                     micro: bool) -> Dict[str, Tensor]:
        """Everything the matcher needs instead of boxes, for the images this process holds: the flat per-image [D, G] tables
        of intersection pixel counts (`mb200_mask_pair_intersections`: ONE launch for all images), their offsets and the
        masks' pixel counts."""
        import numpy as np

        dev = self.device
        if len(self.detection_mask) != len(det_counts) or len(self.groundtruth_mask) != len(gt_counts):
            raise ValueError("every image needs a `masks` entry when `iou_type` contains 'segm'")
        first = lambda c: np.concatenate([[0], np.cumsum(c)])[:-1].astype(np.int64)  # noqa: E731

        def side(entries: List[Tensor], counts: List[int]):
            n = np.asarray(counts, dtype=np.int64)
            length = np.asarray([int(e.numel()) for e in entries], dtype=np.int64)
            words = np.where(n > 0, (length - 3 - n) // np.maximum(n, 1), 0)
            if np.any(length != 3 + n + n * words):
                raise ValueError("a mask state entry does not match the number of labels of its image")
            base = first(length)
            img = np.repeat(np.arange(len(counts)), n)
            k = np.arange(int(n.sum())) - np.repeat(first(n), n)
            flat = torch.cat(entries) if entries else torch.zeros(0, dtype=torch.int32, device=dev)
            area_index = torch.from_numpy(base[img] + 3 + k).to(dev)
            word_off = torch.from_numpy(base[img] + 3 + n[img] + k * words[img]).to(dev)
            return n, words, flat, flat[area_index].to(torch.float64), word_off, base

        dn, dwords, dflat, det_area, det_word_off, dbase = side(self.detection_mask, det_counts)
        gn, gwords, gflat, gt_area, gt_word_off, gbase = side(self.groundtruth_mask, gt_counts)
        both = np.nonzero((dn > 0) & (gn > 0))[0]
        if both.size:  # (H, W) of the two sides of an image, from the entries' headers: one device comparison
            hw = lambda flat, base: flat[torch.from_numpy(np.stack([base[both] + 1, base[both] + 2], 1)).to(dev)]  # noqa: E731
            if np.any(dwords[both] != gwords[both]) or not bool(torch.equal(hw(dflat, dbase), hw(gflat, gbase))):
                raise ValueError("the masks of the predictions and of the target of one image must have the same height and width")
        pairs = dn * gn
        to_dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).astype(dt)).to(dev)  # noqa: E731
        pair_off = to_dev(first(pairs), np.int64)
        inter = _native.mask_pair_intersections(
            dflat, det_word_off, gflat, gt_word_off, to_dev(np.concatenate([[0], np.cumsum(dn)]), np.int32),
            to_dev(np.concatenate([[0], np.cumsum(gn)]), np.int32), to_dev(np.where(dn > 0, dwords, gwords), np.int32),
            det_label, gt_label, micro, pair_off, int(pairs.sum()), int(pairs.max()) if len(pairs) else 0)
        return {"pair_inter": inter, "pair_off": pair_off, "det_area": det_area, "gt_area": gt_area}

    # ------------------------------------------------------------------------------------------------
    # cross-rank sync of the per-image list states
    # ------------------------------------------------------------------------------------------------
    def _sync_states_fast(self, group: Optional[Any]) -> bool:
        """Default-sync fast path (called by ``Metric.sync`` when no ``dist_sync_fn`` was given).

        The reference gathers the ``dist_reduce_fx=None`` list states one per-image tensor at a time — 7 collectives
        (+ barrier + shape gather each) per image, and it dead-locks unless every rank holds the same number of images
        (metric.py:501-540 as reached from detection/mean_ap.py:1031-1043).  Here every rank packs its seven flat arrays
        (plus the bit-packed masks with ``iou_type`` "segm" — the reference ships pickled run-length tuples through
        ``all_gather_object``, :1041-1063) and the per-image counts into ONE byte buffer: two collectives in total (sizes,
        payload), ragged image counts allowed.  Afterwards the states are per-image lists again, images interleaved rank by rank exactly like the
        reference's ``_flatten`` of per-image gathers (image i of rank 0, image i of rank 1, ...).
        """
        from metrics_b200.parallel_sync import _gather_equal

        dist = torch.distributed
        group = group or dist.group.WORLD
        world = dist.get_world_size(group)
        dev = self.device
        boxes, masks = "bbox" in self.iou_type, "segm" in self.iou_type
        n_img = len(self.detection_labels)
        det_counts = [int(t.shape[0]) for t in self.detection_labels]
        gt_counts = [int(t.shape[0]) for t in self.groundtruth_labels]
        n_det, n_gt = sum(det_counts), sum(gt_counts)
        # mask entries are ragged int32 rows (one per image): their lengths travel with the per-image counts
        dm_len = [int(t.numel()) for t in self.detection_mask] if masks else []
        gm_len = [int(t.numel()) for t in self.groundtruth_mask] if masks else []
        if masks and (len(dm_len) != n_img or len(gm_len) != n_img):
            raise ValueError("every image needs a `masks` entry when `iou_type` contains 'segm'")
        # 8-byte fields first so that every field starts 8-byte aligned inside the row
        fields = [
            self._cat_or_empty(self.detection_labels, (0,), torch.int64, dev),
            self._cat_or_empty(self.groundtruth_labels, (0,), torch.int64, dev),
            self._cat_or_empty(self.groundtruth_crowds, (0,), torch.int64, dev),
            self._cat_or_empty(self.groundtruth_area, (0,), torch.float64, dev),
            torch.tensor(det_counts + gt_counts + dm_len + gm_len, dtype=torch.int64, device=dev),
            self._cat_or_empty(self.detection_scores, (0,), torch.float32, dev),
        ]
        if boxes:
            fields += [self._cat_or_empty(self.detection_box, (0, 4), torch.float32, dev),
                       self._cat_or_empty(self.groundtruth_box, (0, 4), torch.float32, dev)]
        if masks:
            fields += [self._cat_or_empty(self.detection_mask, (0,), torch.int32, dev),
                       self._cat_or_empty(self.groundtruth_mask, (0,), torch.int32, dev)]
        payload = torch.cat([f.contiguous().reshape(-1).view(torch.uint8) for f in fields])
        sizes = _gather_equal(torch.tensor([n_img, n_det, n_gt, sum(dm_len), sum(gm_len)], dtype=torch.int64, device=dev),
                              group, world).tolist()
        per_img = 4 if masks else 2
        row_bytes = max(8 * (nd + 3 * ng + per_img * ni) + 4 * nd + (16 * (nd + ng) if boxes else 0) + 4 * (ndm + ngm)
                        for ni, nd, ng, ndm, ngm in sizes)
        row_bytes = (row_bytes + 15) // 16 * 16
        if row_bytes == 0:
            return True
        row = torch.zeros(row_bytes, dtype=torch.uint8, device=dev)
        row[: payload.numel()] = payload
        rows = _gather_equal(row, group, world)

        per_rank = []
        for r, (ni, nd, ng, ndm, ngm) in enumerate(sizes):
            buf, off = rows[r], 0

            def take(count: int, dtype: torch.dtype, width: int = 1) -> Tensor:
                nonlocal off
                nbytes = count * width * torch.empty((), dtype=dtype).element_size()
                out = buf[off:off + nbytes].view(dtype)
                off += nbytes
                return out.reshape(count, width) if width > 1 else out

            det_label, gt_label, gt_crowd, gt_area = take(nd, torch.int64), take(ng, torch.int64), take(ng, torch.int64), take(ng, torch.float64)
            counts = take(per_img * ni, torch.int64).tolist()
            det_score = take(nd, torch.float32)
            dc, gc = counts[:ni], counts[ni:2 * ni]
            entry = {
                "detection_scores": det_score.split(dc), "detection_labels": det_label.split(dc),
                "groundtruth_labels": gt_label.split(gc), "groundtruth_crowds": gt_crowd.split(gc),
                "groundtruth_area": gt_area.split(gc),
            }
            if boxes:
                entry["detection_box"] = take(nd, torch.float32, 4).split(dc)
                entry["groundtruth_box"] = take(ng, torch.float32, 4).split(gc)
            if masks:
                entry["detection_mask"] = take(ndm, torch.int32).split(counts[2 * ni:3 * ni])
                entry["groundtruth_mask"] = take(ngm, torch.int32).split(counts[3 * ni:])
            per_rank.append(entry)
        max_img = max(s[0] for s in sizes)
        for name in per_rank[0]:
            setattr(self, name, [per_rank[r][name][i] for i in range(max_img) for r in range(world) if i < sizes[r][0]])
        return True

    # ------------------------------------------------------------------------------------------------
    # COCO json on either side of the metric (reference :651-825, :867-958)
    # ------------------------------------------------------------------------------------------------
    @staticmethod
    def coco_to_tm(
        coco_preds: str,
        coco_target: str,
        iou_type: Union[Literal["bbox", "segm"], List[str]] = "bbox",
        backend: Literal["pycocotools", "faster_coco_eval"] = "pycocotools",
    ) -> Tuple[List[Dict[str, Tensor]], List[Dict[str, Tensor]]]:
        """COCO ground-truth json (``{"annotations": [...], ...}``) + COCO results json (a list of detections) -> the
        ``(preds, target)`` lists ``update`` takes (reference :651-760).  The files are read directly — the reference goes
        through ``pycocotools.COCO(...).loadRes`` only to get the same annotation lists back.  One entry per image that
        has at least one ground-truth annotation, in order of first appearance; boxes stay in the files' xywh format.
        With "segm", run-length coded segmentations (compressed strings or count lists) become uint8 ``masks``
        (metrics_b200/detection/rle.py); polygon segmentations need pycocotools' rasteriser and raise."""
        kinds = (iou_type,) if isinstance(iou_type, str) else tuple(iou_type)
        if any(k not in ("bbox", "segm") for k in kinds):
            raise ValueError(f"Expected argument `iou_type` to be one of ('bbox', 'segm') or a tuple of, but got {iou_type}")
        boxes, masks = "bbox" in kinds, "segm" in kinds
        with open(coco_target) as fh:
            gt_file = json.load(fh)
        with open(coco_preds) as fh:
            dt_file = json.load(fh)
        if not isinstance(gt_file, dict):
            raise ValueError(f"annotation file format {type(gt_file)} not supported")
        if not isinstance(dt_file, list):
            raise ValueError("results in not an array of objects")
        known_images = {img["id"] for img in gt_file.get("images", [])} or {a["image_id"] for a in gt_file["annotations"]}
        if any(d["image_id"] not in known_images for d in dt_file):
            raise ValueError("Results do not correspond to current coco set")

        import numpy as np

        from metrics_b200.detection.rle import segmentation_to_mask

        sizes = {img["id"]: (int(img.get("height", 0)), int(img.get("width", 0))) for img in gt_file.get("images", [])}

        def mask_of(ann: dict):  # pycocotools `annToMask` for run-length coded segmentations (reference :710, :726)
            return segmentation_to_mask(ann["segmentation"], *sizes.get(ann["image_id"], (0, 0)))

        per_image: Dict[Any, Dict[str, list]] = {}
        for ann in gt_file["annotations"]:
            slot = per_image.setdefault(ann["image_id"], {"g_boxes": [], "g_masks": [], "g_labels": [], "g_crowd": [], "g_area": [],
                                                          "d_boxes": [], "d_masks": [], "d_labels": [], "d_scores": []})
            if boxes:
                slot["g_boxes"].append(ann["bbox"])
            if masks:
                slot["g_masks"].append(mask_of(ann))
            slot["g_labels"].append(ann["category_id"])
            slot["g_crowd"].append(ann["iscrowd"])
            slot["g_area"].append(ann["area"])
        for det in dt_file:
            slot = per_image.get(det["image_id"])
            if slot is not None:  # detections on images without ground truth are not evaluated (reference :736)
                if boxes:
                    slot["d_boxes"].append(det["bbox"])
                if masks:
                    slot["d_masks"].append(mask_of(det))
                slot["d_labels"].append(det["category_id"])
                slot["d_scores"].append(det["score"])
        preds, target = [], []
        for s in per_image.values():
            p = {"scores": torch.tensor(s["d_scores"], dtype=torch.float32), "labels": torch.tensor(s["d_labels"], dtype=torch.int32)}
            t = {"labels": torch.tensor(s["g_labels"], dtype=torch.int32), "iscrowd": torch.tensor(s["g_crowd"], dtype=torch.int32),
                 "area": torch.tensor(s["g_area"], dtype=torch.float32)}
            if boxes:
                p["boxes"] = torch.tensor(s["d_boxes"], dtype=torch.float32)
                t["boxes"] = torch.tensor(s["g_boxes"], dtype=torch.float32)
            if masks:  # uint8 [n, H, W] like the reference (:746, :757); an image without detections gets an empty tensor
                p["masks"] = torch.tensor(np.array(s["d_masks"]), dtype=torch.uint8)
                t["masks"] = torch.tensor(np.array(s["g_masks"]), dtype=torch.uint8)
            preds.append(p)
            target.append(t)
        return preds, target

    def _coco_dataset(self, labels: List[Tensor], boxes: Optional[List[Tensor]], scores: Optional[List[Tensor]] = None,
                      crowds: Optional[List[Tensor]] = None, area: Optional[List[Tensor]] = None,
                      masks: Optional[List[Tensor]] = None) -> Dict[str, list]:
        """The cached per-image states as one COCO dataset dict (reference :867-958, bbox): annotation ids start at 1,
        image ids are the positions in the state lists, ``area`` falls back to ``w * h`` when missing or not positive.
        Every state kind is brought to the host with ONE copy (the reference does one per image and per annotation)."""
        counts = [int(lab.numel()) for lab in labels]

        def host(items: Optional[List[Tensor]], width: int = 1) -> Optional[list]:
            if items is None:
                return None
            kept = [t.reshape(-1, width) if width > 1 else t.reshape(-1) for t in items if t.numel() > 0]
            return torch.cat(kept).cpu().tolist() if kept else []

        for image_id, (lab, box) in enumerate(zip(labels, boxes or [])):
            if box.numel() != 4 * lab.numel():
                raise ValueError(f"Invalid input box of sample {image_id}, element 0 (expected 4 values, got"
                                 f" {box.numel() // max(1, lab.numel())})")
        flat_labels, flat_boxes = host(labels), host(boxes, 4)
        flat_scores, flat_crowds, flat_area = host(scores), host(crowds), host(area)
        images = [{"id": i} for i in range(len(counts))]
        codes: Optional[list] = None
        if masks is not None:  # run-length codes of the bit-packed masks, on the host (reference :897-905, :943-944)
            from metrics_b200.detection.rle import counts_to_string, entry_to_masks, mask_to_counts

            codes = []
            for image_id, entry in enumerate(masks):
                decoded = entry_to_masks(entry.cpu().numpy())
                if decoded.shape[0]:
                    images[image_id]["height"], images[image_id]["width"] = int(decoded.shape[1]), int(decoded.shape[2])
                for m in decoded:
                    codes.append(({"size": [int(m.shape[0]), int(m.shape[1])], "counts": counts_to_string(mask_to_counts(m))},
                                  int(m.sum())))
        annotations = []
        k = 0
        for image_id, count in enumerate(counts):
            for j in range(count):
                label = flat_labels[k]
                box = flat_boxes[k] if flat_boxes is not None else None
                if not isinstance(label, int):
                    raise ValueError(f"Invalid input class of sample {image_id}, element {j}"
                                     f" (expected value of type integer, got type {type(label)})")
                given = flat_area[k] if flat_area is not None else 0
                computed = codes[k][1] if codes is not None else box[2] * box[3]  # mask area as soon as "segm" is in (:923-925)
                ann = {"id": k + 1, "image_id": image_id, "area": given if given > 0 else computed,
                       "category_id": label, "iscrowd": flat_crowds[k] if flat_crowds is not None else 0}
                if box is not None:
                    ann["bbox"] = box
                if codes is not None:
                    ann["segmentation"] = codes[k][0]
                    if box is not None:  # both IoU types: the reference keeps both areas (:926-939)
                        ann["area_bbox"], ann["area_segm"] = box[2] * box[3], codes[k][1]
                if flat_scores is not None:
                    if not isinstance(flat_scores[k], float):
                        raise ValueError(f"Invalid input score of sample {image_id}, element {j}"
                                         f" (expected value of type float, got type {type(flat_scores[k])})")
                    ann["score"] = flat_scores[k]
                annotations.append(ann)
                k += 1
        return {"images": images, "annotations": annotations,
                "categories": [{"id": c, "name": str(c)} for c in self._get_classes()]}

    def tm_to_coco(self, name: str = "tm_map_input") -> None:
        """Write everything ``update`` has cached as ``{name}_preds.json`` (the COCO results list) and
        ``{name}_target.json`` (the COCO ground-truth dataset), reference :762-825.  Masks are written as compressed run-length
        codes (metrics_b200/detection/rle.py) — this is an export path: the bit rows are decoded on the host."""
        with_boxes, with_masks = "bbox" in self.iou_type, "segm" in self.iou_type
        target = self._coco_dataset(self.groundtruth_labels, self.groundtruth_box if with_boxes else None,
                                    crowds=self.groundtruth_crowds, area=self.groundtruth_area,
                                    masks=self.groundtruth_mask if with_masks else None)
        preds = self._coco_dataset(self.detection_labels, self.detection_box if with_boxes else None, scores=self.detection_scores,
                                   masks=self.detection_mask if with_masks else None)
        with open(f"{name}_preds.json", "w") as fh:
            fh.write(json.dumps(preds["annotations"], indent=4))
        with open(f"{name}_target.json", "w") as fh:
            fh.write(json.dumps(target, indent=4))

    def _get_classes(self) -> List[int]:
        if len(self.detection_labels) > 0 or len(self.groundtruth_labels) > 0:
            return torch.cat(self.detection_labels + self.groundtruth_labels).unique().cpu().tolist()
        return []

    @staticmethod
    def _cat_or_empty(items: List[Tensor], shape: Tuple[int, ...], dtype: torch.dtype, device: torch.device) -> Tensor:
        """One flat ``[total, *shape[1:]]`` tensor from the per-image list (empty images contribute nothing)."""
        if not items:
            return torch.empty(shape, dtype=dtype, device=device)
        try:  # common case: every entry already has the right trailing shape -> no per-image Python work
            flat = torch.cat(items)
            if flat.ndim != len(shape) or tuple(flat.shape[1:]) != tuple(shape[1:]):  # e.g. a lone `[1, 0]` "no boxes" entry
                raise RuntimeError("layout mismatch")
        except RuntimeError:
            items = [t.reshape(-1, *shape[1:]) for t in items if t.numel() > 0]
            if not items:
                return torch.empty(shape, dtype=dtype, device=device)
            flat = torch.cat(items)
        return flat.to(dtype)

    def _stats_dict(self, stats: List[Tensor], prefix: str = "") -> Dict[str, Tensor]:
        mdt = self.max_detection_thresholds
        names = ["map", "map_50", "map_75", "map_small", "map_medium", "map_large", f"mar_{mdt[0]}", f"mar_{mdt[1]}",
                 f"mar_{mdt[2]}", "mar_small", "mar_medium", "mar_large"]
        return {prefix + n: s.to(torch.float32).reshape(1) for n, s in zip(names, stats)}

    def _local_states(self) -> Dict[str, Any]:
        """The per-image list states of this process as flat device tensors (+ per-image counts)."""
        dev = self.device
        out: Dict[str, Any] = {
            "det_counts": [int(t.shape[0]) for t in self.detection_labels],
            "gt_counts": [int(t.shape[0]) for t in self.groundtruth_labels],
            "det_score": self._cat_or_empty(self.detection_scores, (0,), torch.float32, dev),
            "det_label": self._cat_or_empty(self.detection_labels, (0,), torch.int64, dev),
            "gt_label": self._cat_or_empty(self.groundtruth_labels, (0,), torch.int64, dev),
            "gt_crowd": self._cat_or_empty(self.groundtruth_crowds, (0,), torch.uint8, dev),
            "gt_area": self._cat_or_empty(self.groundtruth_area, (0,), torch.float64, dev),
        }
        if "bbox" in self.iou_type:
            out["det_box"] = self._cat_or_empty(self.detection_box, (0, 4), torch.float32, dev)
            out["gt_box"] = self._cat_or_empty(self.groundtruth_box, (0, 4), torch.float32, dev)
        else:  # masks only: the matcher never reads the boxes
            out["det_box"] = torch.zeros((out["det_label"].numel(), 4), dtype=torch.float32, device=dev)
            out["gt_box"] = torch.zeros((out["gt_label"].numel(), 4), dtype=torch.float32, device=dev)
        return out

    def _match(self, st: Dict[str, Any], i_type: str, classes: Tensor, micro: bool, tables: Optional[Dict[str, Tensor]]):
        """COCOeval.evaluateImg over this process' images for one IoU type whenever masks are involved (reference :527-547):
        ``tables`` (`_mask_tables`) provides the mask IoUs for "segm" and — reference :917-933 — the annotation area of a
        ground truth without a positive ``area`` is its MASK area for every IoU type as soon as "segm" is among them."""
        gt_area = st["gt_area"]
        if tables is not None:
            gt_area = torch.where(gt_area > 0, gt_area, tables["gt_area"])
        return _native.coco_map_match(
            st["det_box"], st["det_score"], st["det_label"], st["det_counts"], st["gt_box"], st["gt_label"], st["gt_crowd"],
            gt_area, st["gt_counts"], classes, self.iou_thresholds, self.max_detection_thresholds[-1], micro=micro,
            masks=tables if i_type == "segm" else None, gt_area_exact=tables is not None)

    def compute(self) -> Dict[str, Tensor]:
        """Reference :521-598: one evaluation per IoU type (keys prefixed ``bbox_`` / ``segm_`` when there are two)."""
        dev = self.device
        n_img = len(self.detection_labels)
        minus_one = torch.tensor(-1.0, dtype=torch.float64, device=dev)
        classes_list = self._get_classes()
        multi = len(self.iou_type) > 1
        last = self.max_detection_thresholds[-1]
        result: Dict[str, Tensor] = {}
        if n_img == 0:
            for i_type in self.iou_type:
                prefix = f"{i_type}_" if multi else ""
                result.update(self._stats_dict([minus_one] * 12, prefix))
                result[f"{prefix}map_per_class"] = torch.tensor([-1.0], dtype=torch.float32, device=dev)
                result[f"{prefix}mar_{last}_per_class"] = torch.tensor([-1.0], dtype=torch.float32, device=dev)
            result["classes"] = torch.tensor(classes_list, dtype=torch.int32, device=dev)
            return result

        st = self._local_states()
        classes = torch.tensor(classes_list, dtype=torch.int64, device=dev)
        if classes.numel() == 0:  # images without any box at all
            classes = torch.zeros(1, dtype=torch.int64, device=dev)
        micro = self.average == "micro"
        with_masks = "segm" in self.iou_type
        tables: Dict[bool, Dict[str, Tensor]] = {}

        def tables_for(as_micro: bool) -> Optional[Dict[str, Tensor]]:
            if not with_masks:
                return None
            if as_micro not in tables:
                tables[as_micro] = self._mask_tables(st["det_label"], st["gt_label"], st["det_counts"], st["gt_counts"], as_micro)
            return tables[as_micro]

        def run(i_type: str, as_micro: bool):
            if not with_masks:  # boxes only: matching + accumulation behind one call
                return _native.coco_map_evaluate(
                    st["det_box"], st["det_score"], st["det_label"], st["det_counts"], st["gt_box"], st["gt_label"], st["gt_crowd"],
                    st["gt_area"], st["gt_counts"], classes, as_micro, self.iou_thresholds, self.rec_thresholds,
                    self.max_detection_thresholds)
            (cat, rnk, match, ignore), npig, err = self._match(st, i_type, classes, as_micro, tables_for(as_micro))
            k = 1 if as_micro else int(classes.numel())
            precision, recall, scores, _ = _native.coco_map_accumulate(
                cat, st["det_score"], rnk, match, ignore, npig, k, 0, k, len(self.iou_thresholds), self.rec_thresholds,
                self.max_detection_thresholds)
            return precision, recall, scores, err

        for i_type in self.iou_type:
            prefix = f"{i_type}_" if multi else ""
            precision, recall, scores, err = run(i_type, micro)
            if int(err.item()) != 0:
                raise NotImplementedError("metrics_b200: an image holds more ground truths of one class than the matcher can track")
            extras: Dict[str, Tensor] = {}
            if self.extended_summary:
                extras["ious"] = _pairwise_ious(st["det_box"], st["det_score"], st["det_label"], st["det_counts"], st["gt_box"],
                                                st["gt_label"], st["gt_crowd"], st["gt_counts"], classes_list, micro, last,
                                                masks=tables_for(micro) if i_type == "segm" else None)
                extras["precision"] = precision
                extras["recall"] = recall
                extras["scores"] = scores
            per_class = None
            if self.class_metrics:
                per_class = (precision, recall)
                if micro:  # the reference re-evaluates per class with the true labels (:566-569)
                    per_class = run(i_type, False)[:2]
            result.update(self._results(precision, recall, classes_list, extras, per_class, prefix))
        return result

    def _results(self, precision: Tensor, recall: Tensor, classes_list: List[int], extras: Dict[str, Tensor],
                 per_class: Optional[Tuple[Tensor, Tensor]], prefix: str = "") -> Dict[str, Tensor]:
        """The result dict from the accumulated ``precision [T,R,K,A,M]`` / ``recall [T,K,A,M]`` (reference :571-598)."""
        dev = precision.device
        result: Dict[str, Tensor] = {}
        result.update(self._stats_dict(self._summarize(precision, recall), prefix))
        result.update({prefix + k: v for k, v in extras.items()})
        last = self.max_detection_thresholds[-1]
        if per_class is not None:
            m_last = len(self.max_detection_thresholds) - 1
            result[f"{prefix}map_per_class"] = self._masked_mean(per_class[0][:, :, :, 0, m_last], dims=(0, 1)).to(torch.float32)
            result[f"{prefix}mar_{last}_per_class"] = self._masked_mean(per_class[1][:, :, 0, m_last], dims=(0,)).to(torch.float32)
        else:
            result[f"{prefix}map_per_class"] = torch.tensor([-1.0], dtype=torch.float32, device=dev)
            result[f"{prefix}mar_{last}_per_class"] = torch.tensor([-1.0], dtype=torch.float32, device=dev)
        result["classes"] = torch.tensor(classes_list, dtype=torch.int32, device=dev)
        return result

    # ------------------------------------------------------------------------------------------------
    # evaluation sharded over ranks
    # ------------------------------------------------------------------------------------------------
    def _compute_distributed(self) -> Any:
        """``compute()`` under an NCCL group without gathering a single box.

        The reference gathers every rank's per-image lists to every rank and lets every rank evaluate everything
        (mean_ap.py:1032-1063 ``_sync_dist`` + :521-598).  Here the two phases of COCOeval are sharded along their natural axes:
        every rank MATCHES only its own images (`mb200_coco_map_match`, one CTA per image), the per-detection records
        (class, score, rank, match / ignore words: 32 B) are all-gathered and put into the reference's interleaved image order
        (so ties in score break exactly as in the gathered evaluation), every rank ACCUMULATES only its own K / W classes
        (`mb200_coco_map_accumulate`), and the per-class slices of precision / recall are exchanged.  Bit-identical to the
        gather path (`MB200_SHARDED_MAP=0`) and to one GPU fed the interleaved images.  `average="micro"` (one class) and
        `extended_summary` (needs every box everywhere) keep the gather path."""
        dist = torch.distributed
        if not (dist.is_available() and dist.is_initialized()) or os.environ.get("MB200_SHARDED_MAP", "1") == "0":
            return NotImplemented
        if self.dist_sync_fn is not None or self.average == "micro" or self.extended_summary or self.device.type != "cuda":
            return NotImplemented
        if self.distributed_available_fn is not None and not self.distributed_available_fn():
            return NotImplemented
        group = self.process_group or dist.group.WORLD
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        try:
            if world < 2 or dist.get_backend(group) != "nccl":
                return NotImplemented
        except Exception:
            return NotImplemented
        import numpy as np

        from metrics_b200.parallel_sync import _gather_equal
        from metrics_b200.utilities.distributed import gather_all_tensors

        dev = self.device
        st = self._local_states()
        det_counts, det_score = st["det_counts"], st["det_score"]
        # ---- the class list and the image layout of every rank (two small ragged gathers) -------------------------------------
        labels = self.detection_labels + self.groundtruth_labels
        local_labels = torch.cat(labels).to(torch.int64).unique() if labels else torch.zeros(0, dtype=torch.int64, device=dev)
        classes = torch.cat(gather_all_tensors(local_labels, group)).unique()
        classes_list = classes.cpu().tolist()
        counts_all = [c.cpu().tolist() for c in gather_all_tensors(torch.tensor(det_counts, dtype=torch.int64, device=dev), group)]
        if sum(len(c) for c in counts_all) == 0:
            return NotImplemented  # no image anywhere: the generic path produces the reference's "-1 everywhere" result
        if classes.numel() == 0:
            classes = torch.zeros(1, dtype=torch.int64, device=dev)
        k = int(classes.numel())
        bases = np.concatenate([[0], np.cumsum([sum(c) for c in counts_all])])
        offs = [np.concatenate([[0], np.cumsum(c)]) for c in counts_all]
        pieces = [np.arange(bases[r] + offs[r][i], bases[r] + offs[r][i + 1]) for i in range(max(len(c) for c in counts_all))
                  for r in range(world) if i < len(counts_all[r])]
        perm = torch.from_numpy(np.concatenate(pieces).astype(np.int64) if pieces else np.zeros(0, np.int64)).to(dev)
        cpr = (k + world - 1) // world
        lo = min(rank * cpr, k)
        hi = min(lo + cpr, k)
        # masks stay where they are: every rank intersects the masks of its own images only
        tables = (self._mask_tables(st["det_label"], st["gt_label"], det_counts, st["gt_counts"], False)
                  if "segm" in self.iou_type else None)
        multi = len(self.iou_type) > 1
        result: Dict[str, Tensor] = {}
        for i_type in self.iou_type:
            # ---- phase 1 on this rank's images ----------------------------------------------------------------------------------
            records, npig, err = self._match(st, i_type, classes, False, tables)
            dist.all_reduce(npig, group=group)
            dist.all_reduce(err, op=dist.ReduceOp.MAX, group=group)
            if int(err.item()) != 0:
                raise NotImplementedError("metrics_b200: an image holds more ground truths of one class than the matcher can track")
            # ---- records of all ranks, in the interleaved image order of the gathered evaluation ---------------------------------
            cat, rnk, match, ignore = records
            packed = torch.stack([(cat.to(torch.int64) << 32) | rnk.to(torch.int64),
                                  det_score.contiguous().view(torch.int32).to(torch.int64), match, ignore], dim=1)  # [n_local, 4] int64
            allrec = torch.cat(gather_all_tensors(packed, group))[perm]
            # ---- phase 2 on this rank's classes ------------------------------------------------------------------------------------
            precision, recall, scores, _ = _native.coco_map_accumulate(
                (allrec[:, 0] >> 32).to(torch.int32), allrec[:, 1].to(torch.int32).view(torch.float32),
                (allrec[:, 0] & 0xFFFFFFFF).to(torch.int32), allrec[:, 2], allrec[:, 3], npig, k, lo, hi, len(self.iou_thresholds),
                self.rec_thresholds, self.max_detection_thresholds)
            # ---- the class slices of every rank -----------------------------------------------------------------------------------
            t, r_, m = precision.shape[0], precision.shape[1], precision.shape[4]
            slab_p = torch.full((t, r_, cpr, 4, m), -1.0, dtype=torch.float64, device=dev)
            slab_r = torch.full((t, cpr, 4, m), -1.0, dtype=torch.float64, device=dev)
            slab_p[:, :, : hi - lo] = precision[:, :, lo:hi]
            slab_r[:, : hi - lo] = recall[:, lo:hi]
            precision = _gather_equal(slab_p, group, world).permute(1, 2, 0, 3, 4, 5).reshape(t, r_, world * cpr, 4, m)[:, :, :k].contiguous()
            recall = _gather_equal(slab_r, group, world).permute(1, 0, 2, 3, 4).reshape(t, world * cpr, 4, m)[:, :k].contiguous()
            result.update(self._results(precision, recall, classes_list, {}, (precision, recall) if self.class_metrics else None,
                                        f"{i_type}_" if multi else ""))
        return result

    @staticmethod
    def _masked_mean(x: Tensor, dims: Optional[Tuple[int, ...]] = None) -> Tensor:
        """Mean over the entries ``> -1`` (COCOeval._summarize), -1 if there is none."""
        valid = x > -1
        if dims is None:
            cnt = valid.sum()
            tot = torch.where(valid, x, torch.zeros_like(x)).sum()
        else:
            cnt = valid.sum(dim=dims)
            tot = torch.where(valid, x, torch.zeros_like(x)).sum(dim=dims)
        return torch.where(cnt > 0, tot / cnt.clamp(min=1), torch.full_like(tot, -1.0))

    def _summarize(self, precision: Tensor, recall: Tensor) -> List[Tensor]:
        """The 12 COCO statistics (COCOeval.summarize; stat order of reference :632-648)."""
        m_last = len(self.max_detection_thresholds) - 1
        thr = torch.tensor(self.iou_thresholds, dtype=torch.float64)

        def ap(iou: Optional[float] = None, area: int = 0) -> Tensor:
            s = precision[:, :, :, area, m_last]
            if iou is not None:
                sel = (thr == iou).nonzero().flatten().tolist()
                s = s[sel]
            return self._masked_mean(s)

        def ar(area: int = 0, m: int = m_last) -> Tensor:
            return self._masked_mean(recall[:, :, area, m])

        return [ap(), ap(0.5), ap(0.75), ap(area=1), ap(area=2), ap(area=3), ar(m=0), ar(m=1), ar(m=m_last), ar(area=1),
                ar(area=2), ar(area=3)]
