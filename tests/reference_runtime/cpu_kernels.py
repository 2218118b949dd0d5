"""TEST INFRASTRUCTURE ONLY — torch-CPU stand-ins for the wrappers of `metrics_b200._native`.

`sitecustomize.py` installs them (env `MB200_REF_CPU_KERNELS=1`) so that the REFERENCE's own unit tests, which feed CPU
tensors, can exercise everything ABOVE the C-ABI — argument validation, input formatting, state handling, reducers, metric
classes, collections — against scikit-learn, exactly as they test the reference.  The kernels themselves are verified on the
GPU by tests/test_*_gpu.py; nothing here is importable from the product (`metrics_b200` never imports `tests`).

Every function mirrors the contract of the wrapper of the same name in metrics_b200/_native.py.
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor

FLAG_TARGET_RANGE, FLAG_PREDS_RANGE = 1, 2


def launch_count() -> int:
    return 0


def _labels_from(preds: Tensor, target: Tensor):
    """(pred labels, target labels) flattened; class dim of float scores reduced with torch.argmax."""
    if preds.ndim == target.ndim + 1:
        preds = preds.argmax(dim=1)
    return preds.reshape(-1).long(), target.reshape(-1).long()


def _admit(p: Tensor, t: Tensor, num_classes: int, ignore_index: Optional[int], err_flag: Optional[Tensor], int_preds: bool):
    keep = torch.ones_like(t, dtype=torch.bool)
    if ignore_index is not None:
        keep &= t != ignore_index
    bad_t = keep & ((t < 0) | (t >= num_classes))
    bad_p = keep & ((p < 0) | (p >= num_classes)) if int_preds else torch.zeros_like(keep)
    if err_flag is not None:
        if bool(bad_t.any()):
            err_flag |= FLAG_TARGET_RANGE
        if bool(bad_p.any()):
            err_flag |= FLAG_PREDS_RANGE
    keep &= ~bad_t & ~bad_p
    return p[keep], t[keep]


def multiclass_confmat_update_(confmat, preds, target, num_classes, ignore_index, err_flag=None) -> None:
    int_preds = not preds.is_floating_point()
    p, t = _labels_from(preds, target)
    p, t = _admit(p, t, num_classes, ignore_index, err_flag, int_preds)
    confmat += torch.bincount(t * num_classes + p, minlength=num_classes**2).reshape(num_classes, num_classes)


def _per_class_counts(p: Tensor, t: Tensor, num_classes: int):
    cm = torch.bincount(t * num_classes + p, minlength=num_classes**2).reshape(num_classes, num_classes)
    tp = cm.diag()
    fp = cm.sum(0) - tp
    fn = cm.sum(1) - tp
    tn = cm.sum() - (tp + fp + fn)
    return tp, fp, tn, fn


def multiclass_stat_scores_update_(tp, fp, tn, fn, workspace, preds, target, num_classes, ignore_index, micro, err_flag=None) -> None:
    int_preds = not preds.is_floating_point()
    p, t = _labels_from(preds, target)
    p, t = _admit(p, t, num_classes, ignore_index, err_flag, int_preds)
    if micro:
        match = (p == t).sum()
        miss = (p != t).sum()
        tp += match
        fp += miss
        fn += miss
        tn += num_classes * p.numel() - (match + 2 * miss)
        return
    a, b, c, d = _per_class_counts(p, t, num_classes)
    tp += a
    fp += b
    tn += c
    fn += d


def multiclass_stats_softmax_update_(tp, fp, tn, fn, workspace, preds, target, num_classes, micro, err_flag=None) -> Tensor:
    multiclass_stat_scores_update_(tp, fp, tn, fn, workspace, preds, target, num_classes, None, micro, err_flag)
    return softmax_if_logits(preds)


def multiclass_stat_scores_topk_update_(tp, fp, tn, fn, workspace, preds, target, num_classes, top_k, ignore_index, err_flag=None) -> None:
    if preds.ndim != 2 or target.ndim != 1:
        raise NotImplementedError("metrics_b200: top_k > 1 supports `preds` of shape (N, C) with `target` of shape (N,)")
    t = target.long()
    keep = torch.ones_like(t, dtype=torch.bool)
    if ignore_index is not None:
        keep &= t != ignore_index
    bad = keep & ((t < 0) | (t >= num_classes))
    if err_flag is not None and bool(bad.any()):
        err_flag |= FLAG_TARGET_RANGE
    keep &= ~bad
    scores, t = preds[keep].float(), t[keep]
    # k best indices with the lowest index first among equal scores (the kernel's rule)
    order = torch.argsort(-scores, dim=1, stable=True)[:, :top_k]
    in_topk = (order == t[:, None]).any(1)
    p = torch.where(in_topk, t, order[:, 0])
    a, b, c, d = _per_class_counts(p, t, num_classes)
    tp += a
    fp += b
    tn += c
    fn += d


def multiclass_stat_scores_samplewise(preds, target, num_classes, ignore_index, err_flag=None):
    n = target.shape[0]
    p_all = preds.argmax(dim=1) if preds.ndim == target.ndim + 1 else preds
    int_preds = not preds.is_floating_point()
    outs = []
    for i in range(n):
        p, t = p_all[i].reshape(-1).long(), target[i].reshape(-1).long()
        p, t = _admit(p, t, num_classes, ignore_index, err_flag, int_preds)
        outs.append(torch.stack(_per_class_counts(p, t, num_classes)))
    stacked = torch.stack(outs) if outs else torch.zeros((0, 4, num_classes), dtype=torch.long)
    return stacked[:, 0], stacked[:, 1], stacked[:, 2], stacked[:, 3]


def argmax_rows(preds: Tensor) -> Tensor:
    return preds.argmax(dim=1)


def _is_logits(x: Tensor) -> bool:
    return bool(((x < 0) | (x > 1)).any())


def sigmoid_if_logits(preds: Tensor) -> Tensor:
    return preds.sigmoid() if preds.numel() and _is_logits(preds) else preds.clone()


def softmax_if_logits(preds: Tensor) -> Tensor:
    return preds.softmax(1) if preds.numel() and _is_logits(preds) else preds.clone()


def _one_curve(scores: Tensor, positive: Tensor, n_pad: int):
    """Tie-collapsed descending curve of one binary problem: auroc, ap, counts row, padded (fps, tps, thr)."""
    n = scores.numel()
    cmp = scores if scores.dtype == torch.float64 else scores.float()  # float64 scores keep all their bits (64-bit keys)
    order = torch.argsort(cmp, descending=True, stable=True)
    s, y = cmp[order], positive[order].long()
    is_end = torch.ones(n, dtype=torch.bool)
    if n > 1:
        is_end[:-1] = s[1:] != s[:-1]
    idx = torch.nonzero(is_end).flatten()
    tps = torch.cumsum(y, 0)[idx]
    fps = idx + 1 - tps
    P, N = int(y.sum()), int(n - y.sum())
    tp_prev = torch.cat([tps.new_zeros(1), tps[:-1]])
    fp_prev = torch.cat([fps.new_zeros(1), fps[:-1]])
    auroc = float(((fps - fp_prev) * (tps + tp_prev)).sum()) / (2.0 * P * N) if P and N else 0.0
    if P:
        ap = float(((tps - tp_prev).double() / P * (tps.double() / (tps + fps).double())).sum())
    else:
        ap = -0.0
    pad = torch.zeros(n_pad)
    f, t, h = pad.clone(), pad.clone(), torch.zeros(n_pad, dtype=s.dtype)
    f[: idx.numel()], t[: idx.numel()], h[: idx.numel()] = fps.float(), tps.float(), s[idx]
    return auroc, ap, [P, N, int(idx.numel())], f, t, h


def curve_weighted_clf_curve(preds: Tensor, target: Tensor, weights: Tensor, pos_label: int = 1):
    cmp = preds if preds.dtype == torch.float64 else preds.float()
    order = torch.argsort(cmp, descending=True, stable=True)
    s, y, w = cmp[order], (target[order] == pos_label).double(), weights.double()[order]
    is_end = torch.ones(s.numel(), dtype=torch.bool)
    is_end[:-1] = s[1:] != s[:-1]
    idx = torch.nonzero(is_end).flatten()
    return torch.cumsum((1 - y) * w, 0)[idx], torch.cumsum(y * w, 0)[idx], s[idx]


def curve_evaluate(preds: Tensor, target: Tensor, num_classes: int = 1, pos_label: int = 1, want_curve: bool = False,
                   unit_range=None):
    n = target.numel()
    rows = []
    for c in range(num_classes):
        if num_classes == 1:
            rows.append(_one_curve(preds.reshape(-1), target.reshape(-1) == pos_label, n))
        else:
            rows.append(_one_curve(preds[:, c], target == c, n))
    auroc = torch.tensor([r[0] for r in rows], dtype=torch.float32)
    ap = torch.tensor([r[1] for r in rows], dtype=torch.float32)
    counts = torch.tensor([r[2] for r in rows], dtype=torch.int64)
    curve = tuple(torch.stack([r[k] for r in rows]) for k in (3, 4, 5)) if want_curve else None
    return auroc, ap, counts, curve


def curve_evaluate_multilabel(preds: Tensor, target: Tensor, num_labels: int, ignore_index: Optional[int] = None,
                              want_curve: bool = False):
    n = preds.shape[0]
    rows = []
    for l in range(num_labels):
        p, t = preds[:, l], target[:, l]
        if ignore_index is not None:
            keep = t != ignore_index
            p, t = p[keep], t[keep]
        rows.append(_one_curve(p, t == 1, n))
    auroc = torch.tensor([r[0] for r in rows], dtype=torch.float32)
    ap = torch.tensor([r[1] for r in rows], dtype=torch.float32)
    counts = torch.tensor([r[2] for r in rows], dtype=torch.int64)
    curve = tuple(torch.stack([r[k] for r in rows]) for k in (3, 4, 5)) if want_curve else None
    return auroc, ap, counts, curve


def binary_stat_counts(preds, target, num_labels, threshold, ignore_index, samplewise, counts=None, err_flag=None) -> Tensor:
    n_outer = preds.shape[0] if preds.ndim > 0 else 1
    if preds.is_floating_point():
        x = preds
        if preds.numel() and _is_logits(preds):
            x = preds.sigmoid()
        p = (x > threshold).long()
    else:
        p = preds.long()
        if err_flag is not None and bool(((p < 0) | (p > 1)).any()):
            err_flag |= FLAG_PREDS_RANGE
    t = target.long()
    p = p.reshape(n_outer, num_labels, -1)
    t = t.reshape(n_outer, num_labels, -1)
    valid = (t == 0) | (t == 1)
    if ignore_index is not None:
        ignored = t == ignore_index
    else:
        ignored = torch.zeros_like(valid)
    if err_flag is not None and bool((~valid & ~ignored).any()):
        err_flag |= FLAG_TARGET_RANGE
    valid = valid & ~ignored  # ignore_index may itself be 0 or 1
    eq = p == t
    dims = (2,) if samplewise else (0, 2)
    tp = (valid & eq & (t == 1)).sum(dims)
    fp = (valid & ~eq & (t == 0)).sum(dims)
    tn = (valid & eq & (t == 0)).sum(dims)
    fn = (valid & ~eq & (t == 1)).sum(dims)
    out = torch.stack([tp, fp, tn, fn], -1).reshape(-1, 4)
    if counts is None:
        return out
    counts += out
    return counts


_REG_NUM_SUMS = {4: 2, 8: 3, 9: 4}


def regression_sums(preds, target, op, num_outputs=1, param=0.0, eps=0.0) -> Tensor:
    d = int(num_outputs)
    if d < 1 or preds.numel() % d:
        raise ValueError(f"regression_sums: {preds.numel()} elements do not split into rows of num_outputs={d}")
    dtype = torch.promote_types(preds.dtype, target.dtype)
    if not dtype.is_floating_point:
        dtype = torch.float32
    if dtype in (torch.float16, torch.bfloat16):  # half-precision inputs: terms in float32 from the upcast values
        dtype = torch.float32
    p, t = preds.to(dtype).reshape(-1, d), target.to(dtype).reshape(-1, d)
    diff = p - t
    if op == 0:
        terms = [diff * diff]
    elif op == 1:
        terms = [diff.abs()]
    elif op == 2:
        terms = [diff.abs() / t.abs().clamp(min=eps)]
    elif op == 3:
        terms = [diff.abs() / (t.abs() + p.abs()).clamp(min=eps)]
    elif op == 4:
        terms = [diff.abs(), t.abs()]
    elif op == 5:
        terms = [(torch.log1p(p) - torch.log1p(t)) ** 2]
    elif op == 6:
        terms = [torch.log((torch.exp(diff) + torch.exp(-diff)) / 2)]
    elif op == 7:
        terms = [diff.abs() ** param]
    elif op == 8:
        r = t - p
        terms = [t * t, t, r * r]
    elif op == 9:
        r = t - p
        terms = [r, r * r, t, t * t]
    else:  # 10: Tweedie deviance of power `param` + the domain census
        if param == 1:
            dev = 2 * (torch.where(t == 0, torch.zeros_like(t), t * torch.log(t / p)) + p - t)
        elif param == 2:
            dev = 2 * (torch.log(p / t) + t / p - 1)
        else:
            a, b = 1 - param, 2 - param
            dev = 2 * (t.clamp(min=0) ** b / (a * b) - t * p**a / a + p**b / b)
        terms = [dev, (p <= 0).to(p.dtype), (t < 0).to(p.dtype), (t == 0).to(p.dtype)]
    return torch.stack([x.double().sum(0) for x in terms])


def binned_curve_update(preds, target, thresholds, num_classes=1, multilabel=False, ignore_index=None) -> Tensor:
    """`score >= threshold` in the dtype `mb200_binned_curve_compare_dtype` picks: the score dtype above the reference's
    size rule (its loop branch), the promoted dtype below it and for multilabel (its vectorized branch)."""
    n = preds.shape[0] if multilabel else target.numel()
    loop = not multilabel and (n > 50_000 if num_classes == 1 else n * num_classes * num_classes > 1_000_000)
    cmp_dtype = preds.dtype if loop else torch.promote_types(preds.dtype, thresholds.dtype)
    thr = thresholds.to(cmp_dtype)
    t_count = thr.numel()
    if num_classes == 1 and not multilabel:
        p, t = preds.reshape(-1).to(cmp_dtype), target.reshape(-1)
        out = torch.zeros((t_count, 2, 2), dtype=torch.int64)
        ge = p[:, None] >= thr[None, :]
        for y in (0, 1):
            sel = t == y
            out[:, y, 1] = ge[sel].sum(0)
            out[:, y, 0] = sel.sum() - out[:, y, 1]
        return out
    out = torch.zeros((t_count, num_classes, 2, 2), dtype=torch.int64)
    for c in range(num_classes):
        p = preds[:, c].to(cmp_dtype)
        ge = p[:, None] >= thr[None, :]
        for y in (0, 1):
            sel = (target[:, c] == y) if multilabel else ((target == c) == bool(y))
            if multilabel and ignore_index is not None:
                sel &= target[:, c] != ignore_index
            out[:, c, y, 1] = ge[sel].sum(0)
            out[:, c, y, 0] = sel.sum() - out[:, c, y, 1]
    return out


def coco_map_evaluate(det_box, det_score, det_label, det_counts, gt_box, gt_label, gt_crowd, gt_area, gt_counts, classes,
                      micro, iou_thresholds, rec_thresholds, max_dets):
    """Stand-in for the COCO mAP kernels: the numpy oracle (oracle/coco_map.py) on the flat, already-xywh state tensors.
    The GPU tests compare the kernels with that same oracle, so a replay through this stand-in checks only what
    `MeanAveragePrecision.compute` does around the kernel call (concatenation order, counts, defaults, summary table)."""
    import os
    import sys

    root = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    if root not in sys.path:
        sys.path.insert(0, root)
    from oracle.coco_map import coco_evaluate

    def per_image(flat, counts):
        return [piece.numpy() for piece in torch.split(flat, list(counts))]

    res = coco_evaluate(
        per_image(det_box, det_counts), per_image(det_score, det_counts), per_image(det_label, det_counts),
        per_image(gt_box, gt_counts), per_image(gt_label, gt_counts), per_image(gt_crowd, gt_counts),
        per_image(gt_area, gt_counts), box_format="xywh", iou_thresholds=list(iou_thresholds),
        rec_thresholds=list(rec_thresholds), max_detection_thresholds=list(max_dets), average="micro" if micro else "macro")
    as_f64 = lambda name: torch.from_numpy(res[name].astype("float64"))  # noqa: E731
    return as_f64("precision"), as_f64("recall"), as_f64("scores"), torch.zeros(1, dtype=torch.int32)


NAMES = ("launch_count", "multiclass_confmat_update_", "multiclass_stat_scores_update_",
         "multiclass_stat_scores_topk_update_", "multiclass_stat_scores_samplewise", "argmax_rows",
         "sigmoid_if_logits", "softmax_if_logits", "curve_evaluate", "curve_evaluate_multilabel",
         "binary_stat_counts", "regression_sums", "binned_curve_update", "coco_map_evaluate", "curve_weighted_clf_curve",
         "multiclass_stats_softmax_update_", "mask_pack_bits", "mask_pack_entry", "kl_divergence_rows",
         "mask_pair_intersections", "coco_map_match", "coco_map_accumulate")


def mask_pack_bits(masks: Tensor):
    """Stand-in for `mb200_mask_pack_bits`: 32 pixels per int32 word in pixel order (bit k of word w = pixel 32 w + k), areas."""
    n = int(masks.shape[0])
    hw = int(masks[0].numel()) if n else 0
    flat = masks.reshape(n, hw) != 0
    words = (hw + 31) // 32
    pad = torch.zeros((n, words * 32), dtype=torch.int64)
    pad[:, :hw] = flat.to(torch.int64)
    packed = (pad.reshape(n, words, 32) << torch.arange(32, dtype=torch.int64)).sum(2)
    packed = torch.where(packed >= 2 ** 31, packed - 2 ** 32, packed).to(torch.int32)
    return packed, flat.sum(1).to(torch.int64)


def mask_pack_entry(masks: Tensor) -> Tensor:
    """Stand-in for `mb200_mask_pack_entry`: int32 [n, H, W, areas.., bit rows..]."""
    n, h, w = (int(x) for x in masks.shape)
    words, area = mask_pack_bits(masks)
    return torch.cat([torch.tensor([n, h, w], dtype=torch.int32), area.to(torch.int32), words.reshape(-1)])


def _bit_rows(flat: Tensor, word_off: Tensor, words: int):
    """bit rows starting at `word_off` (int32 words, little-endian bit order) -> numpy bool [n, words * 32]"""
    import numpy as np

    rows = np.stack([flat[int(o): int(o) + words].numpy() for o in word_off.tolist()]) if len(word_off) else np.zeros((0, words), np.int32)
    return np.unpackbits(np.ascontiguousarray(rows).view(np.uint8), axis=1, bitorder="little").astype(bool) if words else np.zeros((len(word_off), 0), bool)


def mask_pair_intersections(det_words, det_word_off, gt_words, gt_word_off, det_off, gt_off, img_words, det_label, gt_label,
                            micro, pair_off, n_pairs, max_pairs_per_img) -> Tensor:
    """Stand-in for `mb200_mask_pair_intersections`: per image the [D, G] table of popcount(det & gt), 0 across classes."""
    import numpy as np

    out = np.zeros(max(1, n_pairs), np.float64)
    d_off, g_off = det_off.tolist(), gt_off.tolist()
    for i, words in enumerate(img_words.tolist()):
        d0, d1, g0, g1 = d_off[i], d_off[i + 1], g_off[i], g_off[i + 1]
        if d1 == d0 or g1 == g0:
            continue
        a = _bit_rows(det_words, det_word_off[d0:d1], words).astype(np.int64)
        b = _bit_rows(gt_words, gt_word_off[g0:g1], words).astype(np.int64)
        inter = (a @ b.T).astype(np.float64)
        if not micro:
            inter *= (det_label[d0:d1].numpy()[:, None] == gt_label[g0:g1].numpy()[None, :])
        base = int(pair_off[i])
        out[base: base + inter.size] = inter.reshape(-1)
    return torch.from_numpy(out)


def coco_map_match(det_box, det_score, det_label, det_counts, gt_box, gt_label, gt_crowd, gt_area, gt_counts, classes,
                   iou_thresholds, max_det_last, micro=False, masks=None, gt_area_exact=False):
    """Stand-in for `mb200_coco_map_match(_ex)`: the records of oracle/coco_map.py::match_records as tensors."""
    from oracle.coco_map import match_records

    m = {k: v.numpy() for k, v in masks.items()} if masks is not None else {}
    cat, rank, match, ignore, npig = match_records(
        det_box.numpy(), det_score.numpy(), det_label.numpy(), det_counts, gt_box.numpy(), gt_label.numpy(), gt_crowd.numpy(),
        gt_area.numpy(), gt_counts, classes.numpy(), iou_thresholds, max_det_last, micro=micro, pair_inter=m.get("pair_inter"),
        pair_off=m.get("pair_off"), det_mask_area=m.get("det_area"), gt_mask_area=m.get("gt_area"), gt_area_exact=gt_area_exact)
    as_i64 = lambda x: torch.from_numpy(x.view("int64").copy())  # noqa: E731
    return (torch.from_numpy(cat), torch.from_numpy(rank), as_i64(match), as_i64(ignore)), torch.from_numpy(npig), torch.zeros(1, dtype=torch.int32)


def coco_map_accumulate(det_cat, det_score, det_rank, det_match, det_ignore, npig, num_classes, class_lo, class_hi, n_iou_thr,
                        rec_thresholds, max_dets):
    """Stand-in for `mb200_coco_map_accumulate`: oracle/coco_map.py::accumulate_records on the records."""
    from oracle.coco_map import accumulate_records

    out = accumulate_records(det_cat.numpy(), det_score.numpy(), det_rank.numpy(), det_match.numpy(), det_ignore.numpy(),
                             npig.numpy(), num_classes, class_lo, class_hi, n_iou_thr, rec_thresholds, max_dets)
    return tuple(torch.from_numpy(x) for x in out) + (torch.zeros(1, dtype=torch.int32),)


def kl_divergence_rows(p: Tensor, q: Tensor, log_prob: bool) -> Tensor:
    """Stand-in for `mb200_kl_divergence_rows`: the op chain of functional/regression/kl_divergence.py:25-46 in torch."""
    if log_prob:
        return torch.sum(p.exp() * (p - q), dim=-1)
    p = p / p.sum(dim=-1, keepdim=True)
    q = q / q.sum(dim=-1, keepdim=True)
    res = p * torch.log(p / q)
    return torch.where(p == 0, torch.zeros_like(res), res).sum(dim=-1)


def standins() -> dict:
    """name -> stand-in; a kernel launch is invisible to autograd, so the plain-torch stand-ins are detached the same way."""
    return {name: torch.no_grad()(globals()[name]) for name in NAMES}


def install(native_module) -> None:
    """Replace the kernel wrappers of `metrics_b200._native` by the stand-ins above."""
    for name, fn in standins().items():
        setattr(native_module, name, fn)
