"""CPU: oracle/exact_curves.py (the reference's exact-mode curve chain restated in torch) against goldens from the
unmodified reference (tests/golden/make_golden_exact_curves.py): `_binary_clf_curve` on NaN runs of one label, on runs of
+inf and of -inf, on int64 targets at and above 2^31; binary ROC / PR / AUROC / AP with NaN runs; multilabel with uint8,
int8 and int16 targets whose `ignore_index` wraps in the target's dtype; multiclass with int64 targets 2^32 + c.  Both the
reference's argsort and the documented order (negatives before positives inside NaN / +-inf runs) must reproduce them,
since no golden run mixes labels.  The numpy oracle (oracle/curves.py) must agree on the `_binary_clf_curve` sets too."""
import os

import numpy as np
import pytest
import torch

from oracle import curves as oc
from oracle import exact_curves as oe
from tests.conftest import GOLDEN_DIR


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN_DIR, "exact_curves.npz"), allow_pickle=False)


def names(g, prefix):
    return sorted({k.split("/")[1] for k in g.files if k.startswith(prefix + "/")})


def _t(a):
    return torch.from_numpy(np.array(a))


def _eq(got, want):
    want = _t(want)
    return got.dtype == want.dtype and torch.equal(torch.nan_to_num(got, 7.0), torch.nan_to_num(want, 7.0)) and \
        torch.equal(got.isnan(), want.isnan())


def _preds(g, name):
    p = _t(g[f"clf/{name}/preds"])
    return p.bfloat16() if name.endswith("bfloat16") else p


@pytest.mark.parametrize("documented", [False, True])
def test_binary_clf_curve(golden, documented):
    for name in names(golden, "clf"):
        p, t = _preds(golden, name), _t(golden[f"clf/{name}/target"])
        fps, tps, thr = oe.binary_clf_curve(p, t, documented_order=documented)
        assert _eq(fps, golden[f"clf/{name}/fps"]) and _eq(tps, golden[f"clf/{name}/tps"]), name
        want_thr = _t(golden[f"clf/{name}/thr"])
        assert _eq(thr.float() if thr.dtype == torch.bfloat16 else thr, want_thr.numpy()), name


def test_numpy_oracle_orders_nan_first(golden):
    for name in names(golden, "clf"):
        if name.endswith("bfloat16"):
            continue
        p, t = golden[f"clf/{name}/preds"], golden[f"clf/{name}/target"]
        fps, tps, thr = oc.binary_clf_curve(p, t)
        assert np.array_equal(fps, golden[f"clf/{name}/fps"].astype(np.int64)), name
        assert np.array_equal(tps, golden[f"clf/{name}/tps"].astype(np.int64)), name
        assert np.array_equal(thr, golden[f"clf/{name}/thr"], equal_nan=True), name


def test_binary_computes_with_nan_runs(golden):
    for name in names(golden, "bin"):
        p, t = _t(golden[f"clf/{name}/preds"]), _t(golden[f"clf/{name}/target"])
        p, t = oe.binary_format(p, t)
        fps, tps, thr = oe.binary_clf_curve(p, t, documented_order=True)
        for k, v in zip(("fpr", "tpr", "thr"), oe.binary_roc(fps, tps, thr)):
            assert _eq(v, golden[f"bin/{name}/roc_{k}"]), (name, k)
        for k, v in zip(("p", "r", "thr"), oe.binary_pr(fps, tps, thr, t)):
            assert _eq(v, golden[f"bin/{name}/prc_{k}"]), (name, k)
        assert _eq(oe.binary_auroc(fps, tps, thr), golden[f"bin/{name}/auroc"]), name
        assert _eq(oe.binary_average_precision(fps, tps, thr, t), golden[f"bin/{name}/ap"]), name


def test_multilabel_wrapped_ignore_index(golden):
    for name in names(golden, "ml"):
        p, t = _t(golden[f"ml/{name}/preds"]), _t(golden[f"ml/{name}/target"])
        ign = int(golden[f"ml/{name}/ignore"])
        p, t = oe.multilabel_format(p, t, 3)
        for i, (pi, ti) in enumerate(oe.multilabel_columns(p, t, 3, ign)):
            fps, tps, thr = oe.binary_clf_curve(pi, ti, documented_order=True)
            for k, v in zip(("fpr", "tpr", "thr"), oe.binary_roc(fps, tps, thr)):
                assert _eq(v, golden[f"ml/{name}/roc_{k}{i}"]), (name, i, k)
            for k, v in zip(("p", "r", "thr"), oe.binary_pr(fps, tps, thr, ti)):
                assert _eq(v, golden[f"ml/{name}/prc_{k}{i}"]), (name, i, k)
            assert _eq(oe.binary_auroc(fps, tps, thr), golden[f"ml/{name}/auroc"][i]), (name, i)
            assert _eq(oe.binary_average_precision(fps, tps, thr, ti), golden[f"ml/{name}/ap"][i]), (name, i)


def test_multiclass_int64_targets_beyond_int32(golden):
    p, t = _t(golden["mc/big/preds"]), _t(golden["mc/big/target"])
    assert int(t.max()) >= 2**32
    p, t = oe.multiclass_format(p, t, 4)
    for c in range(4):
        fps, tps, thr = oe.binary_clf_curve(p[:, c], t, pos_label=c, documented_order=True)
        for k, v in zip(("fpr", "tpr", "thr"), oe.binary_roc(fps, tps, thr)):
            assert _eq(v, golden[f"mc/big/roc_{k}{c}"]), (c, k)
        assert _eq(oe.binary_auroc(fps, tps, thr), golden["mc/big/auroc"][c]), c
        assert _eq(oe.binary_average_precision(fps, tps, thr, t == c), golden["mc/big/ap"][c]), c


def test_grouped_counts_match_the_chain():
    g = torch.Generator().manual_seed(3)
    codes = torch.randint(0, 50, (5000,), generator=g)
    pos = torch.rand(5000, generator=g) < 0.3
    fps, tps = oe.grouped_counts(codes, pos, 50, chunk=777)
    f2, t2, _ = oe.binary_clf_curve(1.0 - codes.double() / 64, pos.long())
    assert torch.equal(fps, f2.long()) and torch.equal(tps, t2.long())
    assert oe.auroc_exact(fps, tps) == oc.binary_auroc_exact((1.0 - codes.double() / 64).numpy(), pos.long().numpy())
