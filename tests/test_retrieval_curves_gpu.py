"""GPU: RetrievalAUROC, RetrievalPrecisionRecallCurve and RetrievalRecallAtFixedPrecision (kernels K16e, K16f) against the
reference's goldens and against the exact oracle at the sort and evaluation geometry edges; determinism, the shared group
sort of a compute group and the absence of host reads beyond the group sort's."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import retrieval_curves as orc
from tests import retrieval_curves_cases as rcc
from tests.conftest import GOLDEN_DIR

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _auroc(idx, p, t, top_k=None, max_fpr=None):
    from metrics_b200 import _native

    groups = _native.retrieval_sort(idx.to(DEV), p.to(DEV), t.to(DEV))
    v, e = _native.retrieval_auroc(groups, top_k, max_fpr)
    return v.cpu().numpy(), e.cpu().numpy()


def _curve(idx, p, t, max_k, adaptive_k=False):
    from metrics_b200 import _native

    groups = _native.retrieval_sort(idx.to(DEV), p.to(DEV), t.to(DEV))
    pr, rc, e = _native.retrieval_pr_curve(groups, max_k, adaptive_k)
    return pr.cpu().numpy(), rc.cpu().numpy(), e.cpu().numpy()


def _check_auroc(idx, p, t, top_k=None, max_fpr=None):
    got, empty = _auroc(idx, p, t, top_k, max_fpr)
    want, want_empty = orc.per_query_auroc(idx.numpy(), p.numpy(), t.numpy(), top_k, max_fpr)
    assert np.array_equal(empty, want_empty)
    # the kernel rounds the exact (or float64) area once: within one float32 ulp of the oracle
    spacing = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    ok = (np.abs(got - want) <= spacing) | (np.isnan(got) & np.isnan(want))
    assert ok.all(), (top_k, max_fpr, np.flatnonzero(~ok)[:5], got[~ok][:5], want[~ok][:5])


def _check_curve(idx, p, t, max_k, adaptive_k=False):
    got_p, got_r, empty = _curve(idx, p, t, max_k, adaptive_k)
    want_p, want_r, want_empty = orc.per_query_pr_curve(idx.numpy(), p.numpy(), t.numpy(), max_k, adaptive_k)
    assert np.array_equal(empty, want_empty)
    assert np.array_equal(got_p, want_p), (max_k, adaptive_k, np.argwhere(got_p != want_p)[:5])
    assert np.array_equal(got_r, want_r), (max_k, adaptive_k, np.argwhere(got_r != want_r)[:5])


def test_every_golden_through_classes_and_functionals():
    golden = rcc.load()
    for key, meta in rcc.cases(golden):
        rcc.check_case(golden, key, meta, DEV)


def test_reference_docstring_examples_on_cuda():
    from metrics_b200.functional.retrieval import retrieval_auroc, retrieval_precision_recall_curve
    from metrics_b200.retrieval import RetrievalAUROC, RetrievalPrecisionRecallCurve, RetrievalRecallAtFixedPrecision

    ex = json.load(open(os.path.join(GOLDEN_DIR, "retrieval_curves_surface.json")))["examples"]
    i = torch.tensor([0, 0, 0, 1, 1, 1, 1], device=DEV)
    p = torch.tensor([0.2, 0.3, 0.5, 0.1, 0.3, 0.5, 0.2], device=DEV)
    t = torch.tensor([False, False, True, False, True, False, True], device=DEV)
    assert float(RetrievalAUROC().to(DEV)(p, t, indexes=i)) == ex["RetrievalAUROC"] == 0.75
    p3, t3 = torch.tensor([0.2, 0.3, 0.5], device=DEV), torch.tensor([True, False, True], device=DEV)
    assert float(retrieval_auroc(p3, t3)) == ex["retrieval_auroc"] == 0.5
    assert [x.tolist() for x in retrieval_precision_recall_curve(p3, t3, max_k=2)] == ex["retrieval_precision_recall_curve"]
    i = torch.tensor([0, 0, 0, 0, 1, 1, 1], device=DEV)
    p = torch.tensor([0.4, 0.01, 0.5, 0.6, 0.2, 0.3, 0.5], device=DEV)
    t = torch.tensor([True, False, False, True, True, False, True], device=DEV)
    got = [x.tolist() for x in RetrievalPrecisionRecallCurve(max_k=4).to(DEV)(p, t, indexes=i)]
    assert got == ex["RetrievalPrecisionRecallCurve"]
    assert np.allclose(got[0], [1, .5, .6667, .5], atol=1e-4) and got[1] == [.5, .5, 1, 1]
    r, k = RetrievalRecallAtFixedPrecision(min_precision=0.8).to(DEV)(p, t, indexes=i)
    assert (float(r), int(k)) == tuple(ex["RetrievalRecallAtFixedPrecision"]) == (0.5, 1)
    assert r.is_cuda and k.is_cuda and r.dtype == torch.float32 and k.dtype == torch.int64


def _power_law(seed):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.cat([torch.tensor([1, 2, 31, 32, 33, 1023, 1024, 1025, 4097, 9000]),
                         (torch.rand(300, generator=g) ** -1.3).long().clamp(max=6000)])
    idx = torch.repeat_interleave(torch.arange(len(lengths)) * 3 - 100, lengths)
    return g, idx[torch.randperm(len(idx), generator=g)]


def test_auroc_across_the_warp_cta_threshold():
    g, idx = _power_law(11)
    n = len(idx)
    p = torch.rand(n, generator=g)
    t = (torch.rand(n, generator=g) < 0.3).long()
    for top_k in (None, 1, 3, 33, 1500):
        for max_fpr in (None, 0.1, 0.5):
            _check_auroc(idx, p, t, top_k, max_fpr)


def test_auroc_tie_runs_cross_the_chunks():
    # few distinct scores: every query's tie runs cross the 32-record (warp) and 512-record (CTA) chunk edges
    g, idx = _power_law(12)
    n = len(idx)
    p = torch.randint(0, 7, (n,), generator=g).float() / 6
    t = (torch.rand(n, generator=g) < 0.4).long()
    for top_k in (None, 700, 5000):
        for max_fpr in (None, 0.05, 0.3, 0.0):
            _check_auroc(idx, p, t, top_k, max_fpr)
    # logits: a vote per slice, and distinct large logits that tie only after the sigmoid
    pl = torch.randint(-3, 4, (n,), generator=g).float() * 9
    _check_auroc(idx, pl, t)
    _check_auroc(idx, pl, t, 40, 0.25)


def test_auroc_nan_signed_zero_and_fractional_targets():
    idx = torch.tensor([0] * 7 + [1] * 6 + [2] * 5)
    p = torch.tensor([0.2, float("nan"), 0.9, 0.0, -0.0, float("nan"), 0.5,
                      -0.0, 0.0, 0.0, 0.7, float("nan"), 0.7,
                      3.0, float("nan"), -2.0, 0.5, 0.5])
    t = torch.tensor([0, 1, 0, 1, 0, 0, 1, 1, 0, 1, 0, 1, 0, 1, 0, 0, 1, 0])
    for max_fpr in (None, 0.5):
        _check_auroc(idx, p, t, None, max_fpr)
        _check_auroc(idx, p, t, 4, max_fpr)
    tf = t.float()
    tf[::3] = 0.5  # neither 0 nor 1; a negative when positive
    _check_auroc(idx, p, tf)
    _check_auroc(idx, p, tf, 3)


def test_curve_across_the_warp_cta_threshold():
    g, idx = _power_law(13)
    n = len(idx)
    p = torch.rand(n, generator=g)
    t = (torch.rand(n, generator=g) < 0.2).long()
    for max_k in (1, 32, 33, 1025, 9001, 20000):
        for adaptive_k in (False, True):
            _check_curve(idx, p, t, max_k, adaptive_k)


def test_short_queries_with_a_long_curve():
    g = torch.Generator().manual_seed(14)
    idx = torch.randint(0, 40, (300,), generator=g)
    p = torch.rand(300, generator=g)
    t = (torch.rand(300, generator=g) < 0.5).long()
    _check_curve(idx, p, t, 100_003, True)
    _check_curve(idx, p, t, 100_003, False)


def test_one_query_larger_than_any_tile():
    g = torch.Generator().manual_seed(15)
    n = (1 << 24) + 77
    idx = torch.full((n,), 3, dtype=torch.long)
    p = torch.randint(0, 1000, (n,), generator=g).float() / 999  # tie runs of ~16 700 records
    t = (torch.rand(n, generator=g) < 0.01).long()
    _check_auroc(idx, p, t)
    _check_auroc(idx, p, t, None, 0.1)
    _check_auroc(idx, p, t, 3_000_000, 0.37)
    _check_curve(idx, p, t, 70_000)


def test_wide_index_two_sort_path_and_non_contiguous_inputs():
    g = torch.Generator().manual_seed(16)
    n = 50_000
    q = torch.randint(0, 700, (n,), generator=g)
    p, t = torch.rand(2 * n, generator=g)[::2], (torch.rand(n, 2, generator=g) < 0.3).long()[:, 1]
    assert not p.is_contiguous() and not t.is_contiguous()
    for idx in (q - 10_000, q * (1 << 40) - (1 << 62), q * 3_000_000_000 + (1 << 62) // 3):
        _check_auroc(idx, p, t, 20)
        _check_auroc(idx, p, t, None, 0.2)
        _check_curve(idx, p, t, 90, True)


def test_determinism_and_several_updates():
    from metrics_b200.retrieval import RetrievalAUROC, RetrievalPrecisionRecallCurve

    g = torch.Generator().manual_seed(17)
    n = 300_000
    idx = torch.randint(0, 200, (n,), generator=g).to(DEV)
    p = (torch.randint(0, 50, (n,), generator=g).float() / 49).to(DEV)
    t = (torch.rand(n, generator=g) < 0.1).long().to(DEV)
    for make in (lambda: RetrievalAUROC(aggregation="mean"), lambda: RetrievalAUROC(max_fpr=0.3),
                 lambda: RetrievalPrecisionRecallCurve(max_k=3000)):
        one, many = make().to(DEV), make().to(DEV)
        one.update(p, t, indexes=idx)
        for s in range(0, n, 70_000):
            many.update(p[s:s + 70_000], t[s:s + 70_000], indexes=idx[s:s + 70_000])
        a = one.compute()
        one._computed = None
        one._group_cache.clear()
        b, c = one.compute(), many.compute()
        for x, y, z in zip(*(v if isinstance(v, tuple) else (v,) for v in (a, b, c))):
            assert torch.equal(x, y) and torch.equal(x, z)


def test_a_collection_sorts_once():
    from metrics_b200 import _native
    from metrics_b200.collections import MetricCollection
    from metrics_b200.retrieval import RetrievalAUROC, RetrievalMAP, RetrievalPrecisionRecallCurve

    g = torch.Generator().manual_seed(18)
    idx = torch.randint(0, 500, (40_000,), generator=g).to(DEV)
    p = torch.rand(40_000, generator=g).to(DEV)
    t = (torch.rand(40_000, generator=g) < 0.1).long().to(DEV)
    groups = _native.retrieval_sort(idx, p, t)
    launches = {}
    for name, call in (("map", lambda: _native.retrieval_evaluate(groups, _native.RET_AP)),
                       ("auroc", lambda: _native.retrieval_auroc(groups)),
                       ("curve", lambda: _native.retrieval_pr_curve(groups, 50))):
        before = _native.launch_count()
        call()
        launches[name] = _native.launch_count() - before
    m = RetrievalMAP().to(DEV)
    m.update(p, t, indexes=idx)
    before = _native.launch_count()
    m.compute()
    sort_launches = _native.launch_count() - before - launches["map"]
    alone = {}
    for name, mk in (("map", RetrievalMAP), ("auroc", RetrievalAUROC), ("curve", lambda: RetrievalPrecisionRecallCurve(max_k=50))):
        x = mk().to(DEV)
        x.update(p, t, indexes=idx)
        alone[name] = x.compute()
    coll = MetricCollection({"map": RetrievalMAP(), "auroc": RetrievalAUROC(),
                             "curve": RetrievalPrecisionRecallCurve(max_k=50)}).to(DEV)
    coll.update(p, t, indexes=idx)
    before = _native.launch_count()
    out = coll.compute()
    assert _native.launch_count() - before == sort_launches + sum(launches.values())
    assert torch.equal(out["map"], alone["map"]) and torch.equal(out["auroc"], alone["auroc"])
    assert all(torch.equal(a, b) for a, b in zip(out["curve"], alone["curve"]))


def test_no_host_read_beyond_the_group_sort():
    from metrics_b200.retrieval import RetrievalAUROC, RetrievalPrecisionRecallCurve, RetrievalRecallAtFixedPrecision

    g = torch.Generator().manual_seed(19)
    idx = torch.randint(0, 300, (20_000,), generator=g).to(DEV)
    p = (torch.rand(20_000, generator=g) * 4 - 2).to(DEV)
    t = (torch.rand(20_000, generator=g) < 0.2).long().to(DEV)
    for m in (RetrievalAUROC(), RetrievalAUROC(top_k=10, max_fpr=0.2), RetrievalPrecisionRecallCurve(max_k=64),
              RetrievalRecallAtFixedPrecision(0.3, max_k=64)):
        m = m.to(DEV)
        m.update(p, t, indexes=idx)
        m._groups()  # the group sort and its two reads
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            m.compute()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    # max_k=None reads the longest query's length once
    m = RetrievalPrecisionRecallCurve().to(DEV)
    m.update(p, t, indexes=idx)
    m._groups()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with pytest.warns(UserWarning) as record:
            prec, _, top_k = m.compute()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert sum("synchroniz" in str(w.message) for w in record) == 1
    assert top_k[-1] == int(torch.unique(idx, return_counts=True)[1].max())


def test_max_fpr_above_one_raises_value_error_at_compute():
    from metrics_b200.retrieval import RetrievalAUROC

    m = RetrievalAUROC(max_fpr=2.0).to(DEV)
    m.update(torch.rand(4, device=DEV), torch.tensor([0, 1, 0, 1], device=DEV), indexes=torch.zeros(4, dtype=torch.long, device=DEV))
    with pytest.raises(ValueError, match="`max_fpr` must be 1 or lie in"):
        m.compute()


def test_boundary_ties_follow_arrival_order():
    from metrics_b200.functional.retrieval import retrieval_auroc, retrieval_precision_recall_curve

    # three tied scores, top_k = 2: the first two to arrive enter the slice
    p = torch.tensor([0.5, 0.5, 0.5, 0.1], device=DEV)
    assert float(retrieval_auroc(p, torch.tensor([1, 0, 1, 0], device=DEV), top_k=2)) == 0.5  # one tie group {1, 0}
    assert float(retrieval_auroc(p, torch.tensor([1, 1, 0, 0], device=DEV), top_k=2)) == 0.0  # no negative in the slice
    pr, _, _ = retrieval_precision_recall_curve(p, torch.tensor([0, 1, 1, 0], device=DEV), max_k=1)
    assert pr.tolist() == [0.0]
