"""Panoptic quality states, two independent restatements of the reference's update (functional/detection/
_panoptic_quality_common.py:175-444) that kernel K18 is held to.

`update` (numpy) is the oracle: per image, the three area tables by `np.unique`, then the matching rules vectorised over the
pairs.  `chain_update` (torch, any device) is the same computation as a chain of torch ops — three `torch.unique(dim=0)`
per image, like the reference — and is the benchmark's "chain" arm.  Both divide as the reference does: each int64 operand
rounded to float32, then one IEEE float32 division (what torch's true division of two int64 tensors gives).

Both return ``(iou_sum float64 [K], tp, fp, fn int32 [K])`` of one batch, per-image results summed in image order."""
from __future__ import annotations

import numpy as np
import torch


def categories(things, stuffs):
    """(sorted category ids, their continuous ids, number of things): things in ascending order, then stuffs."""
    order = sorted(things) + sorted(stuffs)
    cid = {c: i for i, c in enumerate(order)}
    ids = sorted(cid)
    return np.array(ids, dtype=np.int64), np.array([cid[c] for c in ids], dtype=np.int64), len(things)


def _colors(x, ids, cids, n_things):
    """[P, 2] (category, instance) -> (continuous id, kept instance); unknown categories -> (K, 0), stuffs -> instance 0."""
    k = len(ids)
    cat, inst = x[:, 0].astype(np.int64), x[:, 1].astype(np.int64)
    pos = np.clip(np.searchsorted(ids, cat), 0, k - 1)
    cid = np.where(ids[pos] == cat, cids[pos], k)
    return cid, np.where(cid < n_things, inst, 0)


def f32_ratio(a, b):
    """float32(a) / float32(b), IEEE round to nearest."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.asarray(a, dtype=np.int64).astype(np.float32) / np.asarray(b, dtype=np.int64).astype(np.float32)


def update_image(p, t, ids, cids, n_things, modified=False):
    """One image: ``p``, ``t`` [P, 2] integer arrays -> (iou_sum float64 [K], tp, fp, fn int64 [K])."""
    k = len(ids)
    iou_sum = np.zeros(k, np.float64)
    tp, fp, fn = (np.zeros(k, np.int64) for _ in range(3))
    if len(p) == 0:
        return iou_sum, tp, fp, fn
    pc, pi = _colors(p, ids, cids, n_things)
    tc, ti = _colors(t, ids, cids, n_things)
    pu, pinv, parea = np.unique(np.stack([pc, pi], 1), axis=0, return_inverse=True, return_counts=True)
    tu, tinv, tarea = np.unique(np.stack([tc, ti], 1), axis=0, return_inverse=True, return_counts=True)
    pinv, tinv = pinv.reshape(-1), tinv.reshape(-1)
    pairs, inter = np.unique(pinv.astype(np.int64) * len(tu) + tinv, return_counts=True)
    ps, ts = pairs // len(tu), pairs % len(tu)
    p_void, t_void = pu[:, 0] == k, tu[:, 0] == k
    pvoid, tvoid = np.zeros(len(pu), np.int64), np.zeros(len(tu), np.int64)
    pvoid[ps[t_void[ts]]] = inter[t_void[ts]]
    tvoid[ts[p_void[ps]]] = inter[p_void[ps]]
    # pairs of one category whose target is not void
    sel = ~t_void[ts] & (pu[ps, 0] == tu[ts, 0])
    ps, ts, inter = ps[sel], ts[sel], inter[sel]
    union = parea[ps] - pvoid[ps] + tarea[ts] - tvoid[ts] - inter
    iou = f32_ratio(inter, union)
    c = tu[ts, 0]
    mstuff = modified & (c >= n_things)
    match = ~mstuff & (iou > np.float32(0.5))
    np.add.at(iou_sum, c[match], iou[match].astype(np.float64))
    np.add.at(tp, c[match], 1)
    np.add.at(iou_sum, c[mstuff & (iou > 0)], iou[mstuff & (iou > 0)].astype(np.float64))
    pmatched, tmatched = np.zeros(len(pu), bool), np.zeros(len(tu), bool)
    pmatched[ps[match]], tmatched[ts[match]] = True, True
    for u, matched, vd, area, out in ((pu, pmatched, pvoid, parea, fp), (tu, tmatched, tvoid, tarea, fn)):
        cand = (u[:, 0] < k) & ~matched & ~(modified & (u[:, 0] >= n_things))
        cand &= f32_ratio(vd, area) <= np.float32(0.5)
        np.add.at(out, u[cand, 0], 1)
    if modified:
        stuff = (tu[:, 0] >= n_things) & (tu[:, 0] < k)
        np.add.at(tp, tu[stuff, 0], 1)
    return iou_sum, tp, fp, fn


def update(preds, target, things, stuffs, modified=False):
    """One batch: ``preds``, ``target`` integer arrays [B, *spatial, 2] -> (iou_sum float64 [K], tp, fp, fn int32 [K])."""
    ids, cids, n_things = categories(things, stuffs)
    k = len(ids)
    preds, target = np.asarray(preds), np.asarray(target)
    b, pixels = preds.shape[0], int(np.prod(preds.shape[1:-1]))
    p, t = preds.reshape(b, pixels, 2), target.reshape(b, pixels, 2)
    iou_sum = np.zeros(k, np.float64)
    counts = [np.zeros(k, np.int64) for _ in range(3)]
    for i in range(b):
        r = update_image(p[i], t[i], ids, cids, n_things, modified)
        iou_sum = iou_sum + r[0]
        counts = [a + x for a, x in zip(counts, r[1:])]
    return (iou_sum, *[x.astype(np.int32) for x in counts])


def compute(iou_sum, tp, fp, fn):
    """(pq, sq, rq, pq_avg, sq_avg, rq_avg) as torch tensors, by the reference's formulas and promotions."""
    iou_sum, tp, fp, fn = (torch.as_tensor(np.asarray(x)) for x in (iou_sum, tp, fp, fn))
    sq = torch.where(tp > 0.0, iou_sum / tp, 0.0)
    den = tp + 0.5 * fp + 0.5 * fn
    rq = torch.where(den > 0.0, tp / den, 0.0)
    pq = sq * rq
    return pq, sq, rq, pq[den > 0].mean(), sq[den > 0].mean(), rq[den > 0].mean()


# ---- torch chain --------------------------------------------------------------------------------------------------------
def _chain_colors(x, ids, cids, n_things):
    k = ids.numel()
    cat, inst = x[:, 0].long().contiguous(), x[:, 1].long()
    pos = torch.searchsorted(ids, cat).clamp(max=k - 1)
    cid = torch.where(ids[pos] == cat, cids[pos], k)
    return torch.stack([cid, torch.where(cid < n_things, inst, 0)], 1)


def chain_update(preds, target, things, stuffs, modified=False):
    """`update` as torch ops on the inputs' device (three ``torch.unique(dim=0)`` per image)."""
    ids_np, cids_np, n_things = categories(things, stuffs)
    dev = preds.device
    ids, cids = torch.from_numpy(ids_np).to(dev), torch.from_numpy(cids_np).to(dev)
    k = ids.numel()
    b, pixels = preds.shape[0], int(np.prod(preds.shape[1:-1]))
    p, t = preds.reshape(b, pixels, 2), target.reshape(b, pixels, 2)
    iou_sum = torch.zeros(k, dtype=torch.float64, device=dev)
    tp, fp, fn = (torch.zeros(k, dtype=torch.int32, device=dev) for _ in range(3))
    for i in range(b):
        if p.shape[1] == 0:
            continue
        pcol, tcol = _chain_colors(p[i], ids, cids, n_things), _chain_colors(t[i], ids, cids, n_things)
        pu, pinv, parea = torch.unique(pcol, dim=0, return_inverse=True, return_counts=True)
        tu, tinv, tarea = torch.unique(tcol, dim=0, return_inverse=True, return_counts=True)
        pairs, inter = torch.unique(torch.stack([pinv, tinv], 1), dim=0, return_counts=True)
        ps, ts = pairs[:, 0], pairs[:, 1]
        p_void, t_void = pu[:, 0] == k, tu[:, 0] == k
        pvoid = torch.zeros(len(pu), dtype=torch.int64, device=dev).index_put_((ps[t_void[ts]],), inter[t_void[ts]])
        tvoid = torch.zeros(len(tu), dtype=torch.int64, device=dev).index_put_((ts[p_void[ps]],), inter[p_void[ps]])
        sel = ~t_void[ts] & (pu[ps, 0] == tu[ts, 0])
        ps, ts, inter = ps[sel], ts[sel], inter[sel]
        iou = inter / (parea[ps] - pvoid[ps] + tarea[ts] - tvoid[ts] - inter)  # int64 / int64: float32
        c = tu[ts, 0]
        mstuff = (c >= n_things) & modified
        match = ~mstuff & (iou > 0.5)
        img_iou = torch.zeros(k, dtype=torch.float64, device=dev)
        img_iou.index_add_(0, c[match], iou[match].double())
        img_iou.index_add_(0, c[mstuff & (iou > 0)], iou[mstuff & (iou > 0)].double())
        img_tp = torch.zeros(k, dtype=torch.int32, device=dev).index_add_(0, c[match], torch.ones_like(c[match], dtype=torch.int32))
        pmatched = torch.zeros(len(pu), dtype=torch.bool, device=dev).index_fill_(0, ps[match], True)
        tmatched = torch.zeros(len(tu), dtype=torch.bool, device=dev).index_fill_(0, ts[match], True)
        img_fp_fn = []
        for u, matched, vd, area in ((pu, pmatched, pvoid, parea), (tu, tmatched, tvoid, tarea)):
            cand = (u[:, 0] < k) & ~matched & ~((u[:, 0] >= n_things) & modified) & (vd / area <= 0.5)
            img_fp_fn.append(torch.bincount(u[cand, 0], minlength=k).int())
        if modified:
            stuff = (tu[:, 0] >= n_things) & (tu[:, 0] < k)
            img_tp += torch.bincount(tu[stuff, 0], minlength=k).int()
        iou_sum += img_iou
        tp += img_tp
        fp += img_fp_fn[0]
        fn += img_fp_fn[1]
    return iou_sum, tp, fp, fn
