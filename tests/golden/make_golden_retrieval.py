"""Generate tests/golden/retrieval.npz and tests/golden/retrieval_surface.json from the UNMODIFIED reference
(TorchMetrics under /root/reference), CPU tensors.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_retrieval.py

Same import set-up as make_golden_segmentation.py.  Every case feeds one or more batches through a reference class and
stores the inputs, `compute()` with the case's aggregation, the per-query values (`compute()` with an identity callable
aggregation, after the empty-query action) and the functional on every query.  Scores are distinct within a query except
in the NDCG tie cases and the NaN cases (one NaN per query outside NDCG).  The json holds the public surface, the state
registry and the reference's errors for invalid arguments; `ret_surface` / `ret_states` also run on this package in
tests/test_retrieval_surface.py.
"""
from __future__ import annotations

import importlib
import inspect
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
CLASSES = ("RetrievalMAP", "RetrievalMRR", "RetrievalPrecision", "RetrievalRecall", "RetrievalHitRate", "RetrievalFallOut",
           "RetrievalRPrecision", "RetrievalNormalizedDCG")
FUNCTIONALS = ("retrieval_average_precision", "retrieval_reciprocal_rank", "retrieval_precision", "retrieval_recall",
               "retrieval_hit_rate", "retrieval_fall_out", "retrieval_r_precision", "retrieval_normalized_dcg")
KIND = dict(zip(CLASSES, ("map", "mrr", "precision", "recall", "hit_rate", "fall_out", "r_precision", "ndcg")))
OUT_OF_SCOPE = ("RetrievalAUROC", "RetrievalPrecisionRecallCurve", "RetrievalRecallAtFixedPrecision", "retrieval_auroc",
                "retrieval_precision_recall_curve")
ATTRS = ("higher_is_better", "is_differentiable", "full_state_update")
CHECKS = ("_check_retrieval_inputs", "_check_retrieval_functional_inputs", "_check_retrieval_target_and_prediction_types")


def _signature(fn):
    sig = inspect.signature(fn)
    return [[n, "<required>" if p.default is inspect.Parameter.empty else repr(p.default)] for n, p in sig.parameters.items()
            if n != "self"]


def ret_surface(pkg: str) -> dict:
    mod = importlib.import_module(f"{pkg}.retrieval")
    fmod = importlib.import_module(f"{pkg}.functional.retrieval")
    chk = importlib.import_module(f"{pkg}.utilities.checks")
    out = {"retrieval.__all__": sorted(n for n in mod.__all__ if n not in OUT_OF_SCOPE),
           "functional.retrieval.__all__": sorted(n for n in fmod.__all__ if n not in OUT_OF_SCOPE)}
    base = importlib.import_module(f"{pkg}.retrieval.base")
    for name in (*CLASSES, "RetrievalMetric"):
        cls = getattr(mod, name, None) or getattr(base, name)
        out[f"retrieval.{name}"] = {"init": _signature(cls.__init__), "update": _signature(cls.update),
                                    "compute": _signature(cls.compute), "attrs": {a: repr(getattr(cls, a, None)) for a in ATTRS}}
    out["retrieval.base._retrieval_aggregate"] = _signature(base._retrieval_aggregate)
    for name in FUNCTIONALS:
        out[f"functional.retrieval.{name}"] = _signature(getattr(fmod, name))
    for name in CHECKS:
        out[f"utilities.checks.{name}"] = _signature(getattr(chk, name))
    return out


def ret_states(pkg: str) -> dict:
    mod = importlib.import_module(f"{pkg}.retrieval")
    out = {}
    for name in CLASSES:
        m = getattr(mod, name)()
        out[name] = {k: {"default": "list" if isinstance(v, list) else [list(v.shape), str(v.dtype)],
                         "reduce": getattr(m._reductions[k], "__name__", None) if m._reductions[k] is not None else None,
                         "persistent": m._persistent[k]} for k, v in m._defaults.items()}
        out[name]["attrs"] = {"empty_target_action": m.empty_target_action, "ignore_index": m.ignore_index,
                              "aggregation": m.aggregation, "allow_non_binary_target": m.allow_non_binary_target}
    return out


def _identity(values, dim=None):
    return values


def _batch(g, q, n_lo, n_hi, idx_base=0, graded=False, float_target=False, nan=False, ties=False, zeros=False):
    """One batch of q queries with n_lo..n_hi documents each, records shuffled across queries."""
    idx, p, t = [], [], []
    for j in range(q):
        n = int(torch.randint(n_lo, n_hi + 1, (1,), generator=g))
        scores = torch.randperm(1000, generator=g)[:n].float() / 997.0  # distinct
        if ties:
            scores = torch.randint(0, 3, (n,), generator=g).float() / 2
        if zeros and n >= 2:  # -0 and +0 tie: only NDCG (tie-averaged) defines the result; elsewhere one -0 alone
            scores[0], scores[1] = (0.0, -0.0) if graded else (-0.0, scores[1])
        if nan and n >= 2:
            scores[int(torch.randint(0, n, (1,), generator=g))] = float("nan")
        if graded:
            tt = torch.randint(-1, 4, (n,), generator=g)
        else:
            tt = (torch.rand(n, generator=g) < 0.3).long()
        if float_target:
            tt = tt.float() * (0.5 if graded else 1.0)
        idx.append(torch.full((n,), idx_base + j * 3 - 7, dtype=torch.long))
        p.append(scores)
        t.append(tt)
    idx, p, t = torch.cat(idx), torch.cat(p), torch.cat(t)
    perm = torch.randperm(len(idx), generator=g)
    return idx[perm], p[perm], t[perm]


def _update_compute(m, p, t, i):
    m.update(p, t, indexes=i)
    return m.compute()


def retrieval_golden():
    from torchmetrics import retrieval as R  # noqa: N812
    from torchmetrics.functional import retrieval as F  # noqa: N812

    g = torch.Generator().manual_seed(1616)
    out, meta = {}, []

    def put(cls, kwargs, batches, aggregation="mean", stable_ties=False):
        key = f"case{len(meta)}"
        m = getattr(R, cls)(aggregation=aggregation, **kwargs)
        mv = getattr(R, cls)(aggregation=_identity, **kwargs)
        for b, (i, p, t) in enumerate(batches):
            m.update(p, t, indexes=i)
            mv.update(p, t, indexes=i)
            out[f"{key}/indexes{b}"], out[f"{key}/preds{b}"], out[f"{key}/target{b}"] = i.numpy(), p.numpy(), t.numpy()
        try:
            out[f"{key}/compute"] = np.array(float(m.compute()))
            out[f"{key}/values"] = np.atleast_1d(mv.compute().numpy())
            err = ""
        except ValueError as e:
            err = str(e)
        # the functional on every query of the concatenated states, ascending index
        fn = getattr(F, FUNCTIONALS[CLASSES.index(cls)])
        fkw = {k: v for k, v in kwargs.items() if k in ("top_k", "adaptive_k")}
        idx = torch.cat([b[0] for b in batches])
        ps, ts = torch.cat([b[1] for b in batches]), torch.cat([b[2] for b in batches])
        fvals = []
        for q in torch.unique(idx):
            sel = idx == q
            tq = ts[sel]
            if kwargs.get("ignore_index") is not None:
                keep = tq != kwargs["ignore_index"]
                fvals.append(float(fn(ps[sel][keep], tq[keep], **fkw)) if keep.any() else float("nan"))
            else:
                fvals.append(float(fn(ps[sel], tq, **fkw)))
        out[f"{key}/functional"] = np.array(fvals)
        meta.append({"cls": cls, "kwargs": kwargs, "aggregation": aggregation, "batches": len(batches), "error": err,
                     "stable_ties": stable_ties})

    kw_top = [{}, {"top_k": 1}, {"top_k": 3}, {"top_k": 50}]
    for cls in CLASSES:
        graded = cls == "RetrievalNormalizedDCG"
        tops = [{}] if cls == "RetrievalRPrecision" else kw_top
        for kw in tops:
            put(cls, kw, [_batch(g, 6, 1, 12, graded=graded)])
        for agg in ("median", "min", "max"):
            put(cls, {}, [_batch(g, 5, 2, 9, graded=graded)], agg)
        for action in ("neg", "pos", "skip", "error"):
            put(cls, {"empty_target_action": action}, [_batch(g, 7, 1, 5, graded=graded)])
        put(cls, {"empty_target_action": "skip"}, [(torch.zeros(3, dtype=torch.long), torch.tensor([.1, .2, .3]),
                                                   torch.tensor([1, 1, 1]) if cls == "RetrievalFallOut" else torch.zeros(3, dtype=torch.long))])
        put(cls, {"ignore_index": -100}, [_batch(g, 5, 3, 9, graded=graded)])
        ii, pp, tt = _batch(g, 5, 3, 9)
        tt[::4] = -100
        put(cls, {"ignore_index": -100}, [(ii, pp, tt)])
        if cls != "RetrievalRPrecision":  # float targets make the reference's R-Precision slice with a float: TypeError
            put(cls, {}, [_batch(g, 5, 2, 9, graded=graded, float_target=True)])
        put(cls, {}, [_batch(g, 4, 2, 8, graded=graded, nan=True), _batch(g, 4, 2, 8, graded=graded, zeros=True, idx_base=2)])
        put(cls, {}, [_batch(g, 3, 2, 8, graded=graded, idx_base=100) for _ in range(3)])
    for kw in ({"adaptive_k": True, "top_k": 50}, {"adaptive_k": True, "top_k": 2}, {"adaptive_k": False, "top_k": 50}):
        put("RetrievalPrecision", kw, [_batch(g, 6, 1, 8)])
    # NDCG: ties, ties with top_k, ties and NaNs together, float graded targets, a [1, -1] query
    for kw in ({}, {"top_k": 2}, {"top_k": 5}):
        put("RetrievalNormalizedDCG", kw, [_batch(g, 6, 2, 12, graded=True, ties=True)])
        put("RetrievalNormalizedDCG", kw, [_batch(g, 4, 3, 10, graded=True, ties=True, nan=True)])
    i, p, t = _batch(g, 3, 3, 6, graded=True, nan=True, ties=True)
    p[:3] = float("nan")
    put("RetrievalNormalizedDCG", {}, [(i, p, t)])
    put("RetrievalNormalizedDCG", {"empty_target_action": "pos"}, [(torch.tensor([5, 5, 6, 6]), torch.tensor([.3, .7, .1, .2]),
                                                                     torch.tensor([1, -1, 2, 0]))])
    put("RetrievalNormalizedDCG", {}, [_batch(g, 5, 2, 9, graded=True, float_target=True, ties=True)])
    # stable ties outside NDCG
    put("RetrievalMAP", {}, [(torch.zeros(4, dtype=torch.long), torch.tensor([.5, .5, .5, .1]), torch.tensor([0, 1, 0, 1]))],
        stable_ties=True)

    # the reference's errors for invalid arguments and inputs
    errors = {}

    def err(name, fn):
        try:
            fn()
        except Exception as e:  # noqa: BLE001
            errors[name] = [type(e).__name__, str(e)]

    p4, t4, i4 = torch.rand(4), torch.tensor([0, 1, 0, 1]), torch.zeros(4, dtype=torch.long)
    for cls in CLASSES:
        err(f"{cls}/empty_target_action", lambda: getattr(R, cls)(empty_target_action="casual"))
        err(f"{cls}/ignore_index", lambda: getattr(R, cls)(ignore_index=1.5))
        err(f"{cls}/aggregation", lambda: getattr(R, cls)(aggregation="sum"))
        if cls != "RetrievalRPrecision":
            err(f"{cls}/top_k_neg", lambda: getattr(R, cls)(top_k=-1))
            err(f"{cls}/top_k_float", lambda: getattr(R, cls)(top_k=1.5))
            err(f"{cls}/top_k_neg_float", lambda: getattr(R, cls)(top_k=-1.5))
        err(f"{cls}/indexes_none", lambda: getattr(R, cls)().update(p4, t4, None))
        err(f"{cls}/shape", lambda: getattr(R, cls)().update(p4, t4[:3], i4))
        err(f"{cls}/indexes_dtype", lambda: getattr(R, cls)().update(p4, t4, i4.int()))
        err(f"{cls}/all_ignored", lambda: getattr(R, cls)(ignore_index=1).update(p4[1::2], t4[1::2], i4[1::2]))
        err(f"{cls}/target_dtype", lambda: getattr(R, cls)().update(p4, t4.to(torch.uint8), i4))
        err(f"{cls}/preds_dtype", lambda: getattr(R, cls)().update(t4, t4, i4))
        err(f"{cls}/non_binary", lambda: getattr(R, cls)().update(p4, t4 * 2, i4))
    err("RetrievalRPrecision/float_target", lambda: _update_compute(R.RetrievalRPrecision(), p4, t4.float(), i4))
    err("retrieval_r_precision/float_target", lambda: F.retrieval_r_precision(p4, t4.float()))
    err("RetrievalPrecision/adaptive_k", lambda: R.RetrievalPrecision(adaptive_k=1))
    for fname in FUNCTIONALS:
        fn = getattr(F, fname)
        err(f"{fname}/shape", lambda: fn(p4, t4[:3]))
        err(f"{fname}/empty", lambda: fn(p4[:0], t4[:0]))
        err(f"{fname}/scalar", lambda: fn(p4[0], t4[0]))
        err(f"{fname}/non_binary", lambda: fn(p4, t4 * 2))
        if fname != "retrieval_r_precision":
            err(f"{fname}/top_k_zero", lambda: fn(p4, t4, top_k=0))
            err(f"{fname}/top_k_neg_float", lambda: fn(p4, t4, top_k=-1.5))
    err("retrieval_precision/adaptive_k", lambda: F.retrieval_precision(p4, t4, adaptive_k=1))
    return out, meta, errors


if __name__ == "__main__":
    import warnings

    warnings.simplefilter("ignore")
    sys.path.insert(0, os.path.join(HERE, "_standins"))
    sys.path.insert(0, "/root/reference/src")
    data, meta, errors = retrieval_golden()
    data["meta"] = np.array(json.dumps(meta))
    path = os.path.join(HERE, "retrieval.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB,", len(meta), "cases")
    surface = {"surface": ret_surface("torchmetrics"), "states": ret_states("torchmetrics"), "errors": errors}
    with open(os.path.join(HERE, "retrieval_surface.json"), "w") as fh:
        json.dump(surface, fh, indent=0, sort_keys=True)
    print("wrote retrieval_surface.json")
