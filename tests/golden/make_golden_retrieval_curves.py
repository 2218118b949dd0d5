"""Generate tests/golden/retrieval_curves.npz and tests/golden/retrieval_curves_surface.json from the UNMODIFIED reference
(TorchMetrics under /root/reference), CPU tensors: RetrievalAUROC, RetrievalPrecisionRecallCurve,
RetrievalRecallAtFixedPrecision and the functionals retrieval_auroc and retrieval_precision_recall_curve.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_retrieval_curves.py

Same import set-up as make_golden_retrieval.py, whose batch maker and surface helpers it uses.  Every case feeds one or
more batches through a reference class and stores the inputs, `compute()` with the case's aggregation, the per-query
values (`compute()` with an identity callable aggregation, after the empty-query action; not for
RecallAtFixedPrecision, whose epilogue needs one curve) and the functional on every query.  Scores are distinct within
a query except where a case makes ties (score ties, +-0, logits that tie only after the sigmoid): ties at the top_k /
max_k boundary are avoided, since the reference's topk leaves their order open.
"""
from __future__ import annotations

import importlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests.golden.make_golden_retrieval import ATTRS, _batch, _identity, _signature  # noqa: E402

CLASSES = ("RetrievalAUROC", "RetrievalPrecisionRecallCurve", "RetrievalRecallAtFixedPrecision")
FUNCTIONALS = ("retrieval_auroc", "retrieval_precision_recall_curve")
FUNCTIONAL = {"RetrievalAUROC": "retrieval_auroc", "RetrievalPrecisionRecallCurve": "retrieval_precision_recall_curve",
              "RetrievalRecallAtFixedPrecision": "retrieval_precision_recall_curve"}


def curves_surface(pkg: str) -> dict:
    mod = importlib.import_module(f"{pkg}.retrieval")
    fmod = importlib.import_module(f"{pkg}.functional.retrieval")
    out = {"retrieval.__all__": sorted(n for n in mod.__all__ if n in CLASSES),
           "functional.retrieval.__all__": sorted(n for n in fmod.__all__ if n in FUNCTIONALS)}
    for name in CLASSES:
        cls = getattr(mod, name)
        out[f"retrieval.{name}"] = {"init": _signature(cls.__init__), "update": _signature(cls.update),
                                    "compute": _signature(cls.compute), "attrs": {a: repr(getattr(cls, a, None)) for a in ATTRS}}
    for name in FUNCTIONALS:
        out[f"functional.retrieval.{name}"] = _signature(getattr(fmod, name))
    return out


def curves_states(pkg: str) -> dict:
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


def _query(idx, scores, target):
    return (torch.full((len(scores),), idx, dtype=torch.long), torch.tensor(scores, dtype=torch.float32), torch.tensor(target))


def _cat(*qs):
    return tuple(torch.cat([q[i] for q in qs]) for i in range(3))


def curves_golden():
    from torchmetrics import retrieval as R  # noqa: N812
    from torchmetrics.functional import retrieval as F  # noqa: N812

    g = torch.Generator().manual_seed(1717)
    out, meta = {}, []

    def put(cls, kwargs, batches, aggregation="mean"):
        key = f"case{len(meta)}"
        agg = {} if cls == "RetrievalRecallAtFixedPrecision" and aggregation == "mean" else {"aggregation": aggregation}
        m = getattr(R, cls)(**agg, **kwargs)
        mv = getattr(R, cls)(aggregation=_identity, **kwargs) if cls != "RetrievalRecallAtFixedPrecision" else None
        for b, (i, p, t) in enumerate(batches):
            m.update(p, t, indexes=i)
            if mv is not None:
                mv.update(p, t, indexes=i)
            out[f"{key}/indexes{b}"], out[f"{key}/preds{b}"], out[f"{key}/target{b}"] = i.numpy(), p.numpy(), t.numpy()
        err = ""
        try:
            res = m.compute()
            if cls == "RetrievalAUROC":
                out[f"{key}/compute"] = np.array(float(res))
                out[f"{key}/values"] = np.atleast_1d(mv.compute().numpy())
            elif cls == "RetrievalPrecisionRecallCurve":
                for name, x in zip(("precision", "recall", "top_k"), res):
                    out[f"{key}/compute_{name}"] = x.numpy()
                pv, rv, _ = mv.compute()
                out[f"{key}/values_precision"], out[f"{key}/values_recall"] = np.atleast_2d(pv.numpy()), np.atleast_2d(rv.numpy())
            else:
                out[f"{key}/compute_recall"], out[f"{key}/compute_k"] = np.array(float(res[0])), np.array(int(res[1]))
        except (ValueError, IndexError) as e:
            err = f"{type(e).__name__}: {e}"
        # the functional on every query of the concatenated states, ascending index
        fn = getattr(F, FUNCTIONAL[cls])
        fkw = {k: v for k, v in kwargs.items() if k in ("top_k", "max_fpr", "max_k", "adaptive_k")}
        idx = torch.cat([b[0] for b in batches])
        ps, ts = torch.cat([b[1] for b in batches]), torch.cat([b[2] for b in batches])
        ii = kwargs.get("ignore_index")
        if ii is not None:
            keep = ts != ii
            idx, ps, ts = idx[keep], ps[keep], ts[keep]
        fvals, fprec, frec, ftop, flen = [], [], [], [], []
        ferr = ""
        try:
            for q in torch.unique(idx):
                sel = idx == q
                if cls == "RetrievalAUROC":
                    fvals.append(float(fn(ps[sel], ts[sel], **fkw)))
                else:
                    pr, rc, tk = fn(ps[sel], ts[sel], **fkw)
                    fprec.append(pr.numpy()), frec.append(rc.numpy()), ftop.append(tk.numpy()), flen.append(len(pr))
        except (ValueError, IndexError) as e:
            ferr = f"{type(e).__name__}: {e}"
        if not ferr:
            if cls == "RetrievalAUROC":
                out[f"{key}/functional"] = np.array(fvals)
            else:
                out[f"{key}/functional_precision"] = np.concatenate(fprec).astype(np.float32)
                out[f"{key}/functional_recall"] = np.concatenate(frec).astype(np.float32)
                out[f"{key}/functional_top_k"] = np.concatenate(ftop).astype(np.int64)
                out[f"{key}/functional_len"] = np.array(flen, dtype=np.int64)
        meta.append({"cls": cls, "kwargs": kwargs, "aggregation": aggregation, "batches": len(batches), "error": err,
                     "functional_error": ferr})

    def batch(q=6, lo=2, hi=12, **kw):
        return _batch(g, q, lo, hi, **kw)

    # --- AUROC ---------------------------------------------------------------------------------------------------------
    for top_k in (None, 1, 3, 50):
        for max_fpr in (None, 0.1, 0.5, 1.0, 0.0):
            put("RetrievalAUROC", {"top_k": top_k, "max_fpr": max_fpr}, [batch(6, 2, 14)])
    for agg in ("median", "min", "max"):
        put("RetrievalAUROC", {}, [batch(5, 3, 9)], agg)
    for action in ("neg", "pos", "skip", "error"):
        put("RetrievalAUROC", {"empty_target_action": action}, [batch(7, 1, 5)])
    put("RetrievalAUROC", {"empty_target_action": "skip"}, [(torch.zeros(3, dtype=torch.long), torch.tensor([.1, .2, .3]),
                                                             torch.zeros(3, dtype=torch.long))])
    ii, pp, tt = batch(5, 3, 9)
    tt[::4] = -100
    put("RetrievalAUROC", {"ignore_index": -100}, [(ii, pp, tt)])
    put("RetrievalAUROC", {}, [batch(3, 2, 8, idx_base=100) for _ in range(3)])
    # targets: bool, int, float (one fractional value: neither 0 nor 1, and a negative after target.int())
    i, p, t = batch(5, 3, 10)
    put("RetrievalAUROC", {}, [(i, p, t.bool())])
    put("RetrievalAUROC", {"max_fpr": 0.5}, [(i, p, t.float())])
    tf = t.float()
    tf[::3] = 0.5
    put("RetrievalAUROC", {}, [(i, p, tf)])
    put("RetrievalAUROC", {"top_k": 3}, [(i, p, tf)])
    # logits that tie only after the sigmoid; score ties; +-0; only positives; only negatives; positives out of top_k
    logits = _cat(_query(0, [17.0, 18.0, 25.0, -3.0, 2.0], [1, 0, 1, 0, 0]),
                  _query(1, [30.0, 40.0, 0.5, -60.0, -70.0, 1.5], [0, 1, 1, 0, 1, 0]),
                  _query(2, [0.5, 0.5, 0.5, 0.2, 0.2, 0.9], [1, 0, 0, 1, 0, 1]),
                  _query(3, [0.0, -0.0, 0.3, 0.0], [1, 0, 0, 1]),
                  _query(4, [0.3, 0.6, 0.9], [1, 1, 1]),
                  _query(5, [0.3, 0.6, 0.9], [0, 0, 0]),
                  _query(6, [0.9, 0.8, 0.7, 0.2, 0.1], [0, 0, 0, 1, 1]))
    for kw in ({}, {"top_k": 4}, {"max_fpr": 0.5}, {"max_fpr": 0.3, "top_k": 4}, {"empty_target_action": "skip"}):
        put("RetrievalAUROC", kw, [logits])
    for kw in ({}, {"max_fpr": 0.2}, {"max_fpr": 0.0}):
        put("RetrievalAUROC", kw, [batch(6, 5, 20, ties=True)])
    # max_fpr above 1: the reference indexes past the ROC curve
    put("RetrievalAUROC", {"max_fpr": 2.0}, [batch(3, 3, 6)])

    # --- PR curve ------------------------------------------------------------------------------------------------------
    for max_k in (None, 1, 4, 40):
        for adaptive_k in (False, True):
            put("RetrievalPrecisionRecallCurve", {"max_k": max_k, "adaptive_k": adaptive_k}, [batch(6, 1, 12)])
    for agg in ("median", "min", "max"):
        put("RetrievalPrecisionRecallCurve", {"max_k": 6}, [batch(5, 2, 9)], agg)
    for action in ("neg", "pos", "skip", "error"):
        put("RetrievalPrecisionRecallCurve", {"empty_target_action": action, "max_k": 5}, [batch(7, 1, 5)])
    for max_k in (None, 3):
        put("RetrievalPrecisionRecallCurve", {"empty_target_action": "skip", "max_k": max_k},
            [(torch.tensor([0, 0, 0, 4, 4]), torch.tensor([.1, .2, .3, .4, .5]), torch.zeros(5, dtype=torch.long))])
    ii, pp, tt = batch(5, 3, 9)
    tt[::4] = -100
    put("RetrievalPrecisionRecallCurve", {"ignore_index": -100, "max_k": 6}, [(ii, pp, tt)])
    put("RetrievalPrecisionRecallCurve", {"max_k": 7}, [batch(3, 2, 8, idx_base=100) for _ in range(3)])
    i, p, t = batch(5, 3, 10)
    put("RetrievalPrecisionRecallCurve", {"max_k": 8}, [(i, p, t.bool())])
    put("RetrievalPrecisionRecallCurve", {"max_k": 8, "adaptive_k": True}, [(i, p, t.float())])
    tf = t.float()
    tf[::3] = 0.5
    put("RetrievalPrecisionRecallCurve", {"max_k": 8}, [(i, p, tf)])

    # --- RecallAtFixedPrecision ----------------------------------------------------------------------------------------
    for min_precision in (0.0, 0.5, 0.8, 1.0):
        for max_k in (None, 5):
            put("RetrievalRecallAtFixedPrecision", {"min_precision": min_precision, "max_k": max_k}, [batch(6, 2, 10)])
    # nothing qualifies: every query's best document is a negative
    put("RetrievalRecallAtFixedPrecision", {"min_precision": 0.9, "max_k": 4},
        [_cat(_query(0, [0.9, 0.5, 0.1], [0, 1, 1]), _query(1, [0.8, 0.7], [0, 1]))])
    # recall ties: the curve stays flat after the last positive; the largest k must win
    put("RetrievalRecallAtFixedPrecision", {"min_precision": 0.2, "max_k": 6},
        [_cat(_query(0, [0.9, 0.5, 0.1, 0.05], [1, 0, 0, 0]), _query(1, [0.8, 0.7, 0.1], [1, 0, 0]))])
    put("RetrievalRecallAtFixedPrecision", {"min_precision": 0.5, "max_k": 4, "adaptive_k": True},
        [_cat(_query(0, [0.9, 0.5], [1, 0]), _query(1, [0.8, 0.7, 0.1], [1, 1, 0]))])
    put("RetrievalRecallAtFixedPrecision", {"min_precision": 0.5, "empty_target_action": "skip"},
        [(torch.zeros(3, dtype=torch.long), torch.tensor([.1, .2, .3]), torch.zeros(3, dtype=torch.long))])

    # --- the reference's docstring examples ----------------------------------------------------------------------------
    doc_i = torch.tensor([0, 0, 0, 1, 1, 1, 1])
    doc_p = torch.tensor([0.2, 0.3, 0.5, 0.1, 0.3, 0.5, 0.2])
    doc_t = torch.tensor([False, False, True, False, True, False, True])
    pr_i = torch.tensor([0, 0, 0, 0, 1, 1, 1])
    pr_p = torch.tensor([0.4, 0.01, 0.5, 0.6, 0.2, 0.3, 0.5])
    pr_t = torch.tensor([True, False, False, True, True, False, True])
    put("RetrievalAUROC", {}, [(doc_i, doc_p, doc_t)])
    put("RetrievalPrecisionRecallCurve", {"max_k": 4}, [(pr_i, pr_p, pr_t)])
    put("RetrievalRecallAtFixedPrecision", {"min_precision": 0.8}, [(pr_i, pr_p, pr_t)])
    examples = {
        "RetrievalAUROC": float(R.RetrievalAUROC()(doc_p, doc_t, indexes=doc_i)),
        "retrieval_auroc": float(F.retrieval_auroc(torch.tensor([0.2, 0.3, 0.5]), torch.tensor([True, False, True]))),
        "RetrievalPrecisionRecallCurve": [x.tolist() for x in R.RetrievalPrecisionRecallCurve(max_k=4)(pr_p, pr_t, indexes=pr_i)],
        "RetrievalRecallAtFixedPrecision": [float(x) for x in
                                            R.RetrievalRecallAtFixedPrecision(min_precision=0.8)(pr_p, pr_t, indexes=pr_i)],
        "retrieval_precision_recall_curve": [x.tolist() for x in F.retrieval_precision_recall_curve(
            torch.tensor([0.2, 0.3, 0.5]), torch.tensor([True, False, True]), max_k=2)],
    }

    # the reference's errors for invalid arguments and inputs
    errors = {}

    def err(name, fn):
        try:
            fn()
        except Exception as e:  # noqa: BLE001
            errors[name] = [type(e).__name__, str(e)]

    p4, t4, i4 = torch.rand(4), torch.tensor([0, 1, 0, 1]), torch.zeros(4, dtype=torch.long)
    for cls in CLASSES:
        c = getattr(R, cls)
        for name, call in error_calls_class(c, p4, t4, i4).items():
            err(f"{cls}/{name}", call)
    for fname in FUNCTIONALS:
        for name, call in error_calls_functional(getattr(F, fname), p4, t4).items():
            err(f"{fname}/{name}", call)
    return out, meta, errors, examples


def error_calls_class(c, p4, t4, i4) -> dict:
    """The invalid arguments and inputs tried on every class (shared with tests/test_retrieval_curves_surface.py)."""
    name = c.__name__
    calls = {
        "empty_target_action": lambda: c(empty_target_action="casual"),
        "ignore_index": lambda: c(ignore_index=1.5),
        "aggregation": lambda: c(aggregation="sum"),
        "indexes_none": lambda: c().update(p4, t4, None),
        "shape": lambda: c().update(p4, t4[:3], i4),
        "indexes_dtype": lambda: c().update(p4, t4, i4.int()),
        "all_ignored": lambda: c(ignore_index=1).update(p4[1::2], t4[1::2], i4[1::2]),
        "target_dtype": lambda: c().update(p4, t4.to(torch.uint8), i4),
        "preds_dtype": lambda: c().update(t4, t4, i4),
        "non_binary": lambda: c().update(p4, t4 * 2, i4),
    }
    if name == "RetrievalAUROC":
        calls.update({"top_k_neg": lambda: c(top_k=-1), "top_k_float": lambda: c(top_k=1.5), "top_k_zero": lambda: c(top_k=0),
                      "max_fpr_int_one": lambda: c(max_fpr=1), "max_fpr_int_two": lambda: c(max_fpr=2),
                      "max_fpr_neg": lambda: c(max_fpr=-0.5), "max_fpr_str": lambda: c(max_fpr="a")})
    else:
        calls.update({"max_k_zero": lambda: c(max_k=0), "max_k_float": lambda: c(max_k=1.5), "max_k_neg": lambda: c(max_k=-2),
                      "adaptive_k": lambda: c(adaptive_k=1)})
    if name == "RetrievalRecallAtFixedPrecision":
        calls.update({"min_precision_int": lambda: c(min_precision=1), "min_precision_big": lambda: c(min_precision=1.5),
                      "min_precision_neg": lambda: c(min_precision=-0.1)})
    return calls


def error_calls_functional(fn, p4, t4) -> dict:
    """The invalid arguments and inputs tried on every functional."""
    calls = {
        "shape": lambda: fn(p4, t4[:3]),
        "empty": lambda: fn(p4[:0], t4[:0]),
        "scalar": lambda: fn(p4[0], t4[0]),
        "non_binary": lambda: fn(p4, t4 * 2),
        "target_dtype": lambda: fn(p4, t4.to(torch.uint8)),
    }
    if fn.__name__ == "retrieval_auroc":
        calls.update({"top_k_neg": lambda: fn(p4, t4, top_k=-1), "top_k_float": lambda: fn(p4, t4, top_k=1.5),
                      "max_fpr_int_one": lambda: fn(p4, t4, max_fpr=1)})
    else:
        calls.update({"max_k_zero": lambda: fn(p4, t4, max_k=0), "max_k_float": lambda: fn(p4, t4, max_k=1.5),
                      "adaptive_k": lambda: fn(p4, t4, adaptive_k=1)})
    return calls


if __name__ == "__main__":
    import warnings

    warnings.simplefilter("ignore")
    sys.path.insert(0, os.path.join(HERE, "_standins"))
    sys.path.insert(0, "/root/reference/src")
    data, meta, errors, examples = curves_golden()
    data["meta"] = np.array(json.dumps(meta))
    path = os.path.join(HERE, "retrieval_curves.npz")
    np.savez_compressed(path, **data)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB,", len(meta), "cases")
    surface = {"surface": curves_surface("torchmetrics"), "states": curves_states("torchmetrics"), "errors": errors,
               "examples": examples}
    with open(os.path.join(HERE, "retrieval_curves_surface.json"), "w") as fh:
        json.dump(surface, fh, indent=0, sort_keys=True)
    print("wrote retrieval_curves_surface.json")
