"""GPU: the retrieval metrics (kernel K16) against the reference's goldens and against the float64 oracle at the sort and
evaluation geometry edges; determinism, the shared group sort of a compute group and the state round trips."""
import numpy as np
import pytest
import torch

from oracle import retrieval as orc
from tests import retrieval_cases as rc

pytestmark = pytest.mark.gpu
DEV = "cuda"
KINDS = {"map": 0, "mrr": 1, "precision": 2, "recall": 3, "hit_rate": 4, "fall_out": 5, "r_precision": 6, "ndcg": 7}


def _values(kind, idx, p, t, top_k=None, adaptive_k=False):
    from metrics_b200 import _native

    groups = _native.retrieval_sort(idx, p, t)
    ideal = _native.retrieval_sort_ideal(groups) if kind == "ndcg" else None
    v, e = _native.retrieval_evaluate(groups, KINDS[kind], top_k, adaptive_k, ideal)
    return v.cpu().numpy(), e.cpu().numpy()


def _check_against_oracle(kind, idx, p, t, top_k=None, adaptive_k=False):
    got, empty = _values(kind, idx.to(DEV), p.to(DEV), t.to(DEV), top_k, adaptive_k)
    want, want_empty = orc.per_query(kind, idx.cpu().numpy(), p.cpu().numpy(), t.cpu().numpy(), top_k, adaptive_k)
    assert len(got) == len(want)
    assert np.array_equal(empty, want_empty)
    assert rc.ulp_close(got, want.astype(np.float32), False), (kind, np.abs(got - want).max())


def test_every_golden_through_classes_and_functionals():
    golden = rc.load()
    for key, meta in rc.cases(golden):
        if meta["stable_ties"]:
            continue
        rc.check_case(golden, key, meta, DEV)


def test_stable_ties():
    from metrics_b200.functional.retrieval import retrieval_average_precision
    from metrics_b200.retrieval import RetrievalMAP

    p, t = torch.tensor([.5, .5, .5, .1], device=DEV), torch.tensor([0, 1, 0, 1], device=DEV)
    assert float(retrieval_average_precision(p, t)) == 0.5
    m = RetrievalMAP().to(DEV)
    m.update(p, t, indexes=torch.zeros(4, dtype=torch.long, device=DEV))
    assert float(m.compute()) == 0.5


def test_one_query_larger_than_any_tile():
    g = torch.Generator().manual_seed(1)
    n = (1 << 24) + 77
    p = torch.rand(n, generator=g)
    t = (torch.rand(n, generator=g) < 0.01).long()
    idx = torch.full((n,), 5, dtype=torch.long)
    for kind, top_k in (("map", None), ("recall", 100_000), ("precision", 12345), ("mrr", None), ("fall_out", 5_000_000)):
        _check_against_oracle(kind, idx, p, t, top_k)
    # NDCG on three score values: tie runs of millions of records cross every tile and chunk
    pt = torch.randint(0, 3, (n,), generator=g).float()
    got, _ = _values("ndcg", idx.to(DEV), pt.to(DEV), t.to(DEV), 3_000_000)
    want = orc.query_value("ndcg", pt.numpy(), t.numpy(), 3_000_000)
    assert np.isclose(got[0], want, rtol=1e-6)


def test_one_document_per_query():
    g = torch.Generator().manual_seed(2)
    n = 20_000
    idx = torch.randperm(n, generator=g) * 7 - 50_000
    p, t = torch.rand(n, generator=g), torch.randint(0, 2, (n,), generator=g)
    for kind in KINDS:
        _check_against_oracle(kind, idx, p, t.float() if kind == "ndcg" else t, 1 if kind == "precision" else None)


@pytest.mark.parametrize("kind", list(KINDS))
def test_power_law_lengths_across_the_warp_cta_threshold(kind):
    g = torch.Generator().manual_seed(3)
    lengths = torch.cat([torch.tensor([1, 2, 31, 32, 33, 1023, 1024, 1025, 4097, 9000]),
                         (torch.rand(300, generator=g) ** -1.3).long().clamp(max=6000)])
    idx = torch.repeat_interleave(torch.arange(len(lengths)) * 3 - 100, lengths)
    perm = torch.randperm(len(idx), generator=g)
    idx = idx[perm]
    n = len(idx)
    if kind == "ndcg":  # ties everywhere: runs cross the 32- and 512-record chunks
        p = torch.randint(0, 20, (n,), generator=g).float() / 4
        t = torch.randint(-1, 4, (n,), generator=g)
        got, empty = _values(kind, idx.to(DEV), p.to(DEV), t.to(DEV), 700)
        want, want_empty = orc.per_query(kind, idx.numpy(), p.numpy(), t.numpy(), 700)
        assert np.array_equal(empty, want_empty) and np.allclose(got, want, rtol=2e-6, atol=1e-7)
        return
    p = torch.rand(n, generator=g)
    t = (torch.rand(n, generator=g) < 0.2).long()
    for top_k in (None, 3, 1500):
        _check_against_oracle(kind, idx, p, t, None if kind == "r_precision" else top_k, kind == "precision")


def test_nan_and_signed_zero_scores():
    p = torch.tensor([0.2, float("nan"), 0.9, 0.0, -0.0, float("nan"), 0.5])
    t = torch.tensor([0, 1, 0, 1, 0, 2, 1])
    idx = torch.tensor([0, 0, 0, 1, 1, 1, 1])
    got, _ = _values("ndcg", idx.to(DEV), p.to(DEV), t.to(DEV))
    want, _ = orc.per_query("ndcg", idx.numpy(), p.numpy(), t.numpy())
    assert np.allclose(got, want, rtol=1e-6)
    tb = t.clamp(max=1)
    _check_against_oracle("mrr", idx, p, tb)
    _check_against_oracle("map", idx, p, tb)


def test_index_range_edges_and_non_contiguous_inputs():
    g = torch.Generator().manual_seed(4)
    n = 50_000
    q = torch.randint(0, 700, (n,), generator=g)
    p, t = torch.rand(2 * n, generator=g)[::2], (torch.rand(n, 2, generator=g) < 0.3).long()[:, 1]
    assert not p.is_contiguous() and not t.is_contiguous()
    for idx in (q - 10_000, q * (1 << 40) - (1 << 62), q * 3_000_000_000 + (1 << 62) // 3, q * 65_536 - 7):
        for kind in ("map", "recall", "ndcg"):
            if kind == "ndcg":
                got, _ = _values(kind, idx.to(DEV), p.to(DEV), t.to(DEV), 10)
                want, _ = orc.per_query(kind, idx.numpy(), p.numpy(), t.numpy(), 10)
                assert np.allclose(got, want, rtol=2e-6)
            else:
                _check_against_oracle(kind, idx, p, t, 10)


def test_determinism_and_several_updates():
    from metrics_b200.retrieval import RetrievalMAP, RetrievalNormalizedDCG

    g = torch.Generator().manual_seed(5)
    idx = torch.randint(0, 2000, (300_000,), generator=g).to(DEV)
    p = torch.rand(300_000, generator=g).to(DEV)
    t = (torch.rand(300_000, generator=g) < 0.1).long().to(DEV)
    for cls in (RetrievalMAP, RetrievalNormalizedDCG):
        one, many = cls(aggregation=rc.identity).to(DEV), cls(aggregation=rc.identity).to(DEV)
        one.update(p, t, indexes=idx)
        for s in range(0, 300_000, 70_000):
            many.update(p[s:s + 70_000], t[s:s + 70_000], indexes=idx[s:s + 70_000])
        a = one.compute()
        one._computed = None
        one._group_cache.clear()
        assert torch.equal(a, one.compute())
        assert torch.equal(a, many.compute())


def test_a_collection_sorts_once():
    from metrics_b200 import _native
    from metrics_b200.collections import MetricCollection
    from metrics_b200.retrieval import RetrievalMAP, RetrievalMRR, RetrievalPrecision

    g = torch.Generator().manual_seed(6)
    idx = torch.randint(0, 500, (40_000,), generator=g).to(DEV)
    p = torch.rand(40_000, generator=g).to(DEV)
    t = (torch.rand(40_000, generator=g) < 0.1).long().to(DEV)
    alone = {}
    launches = {}
    for name, m in (("map", RetrievalMAP()), ("mrr", RetrievalMRR()), ("p10", RetrievalPrecision(top_k=10))):
        m = m.to(DEV)
        m.update(p, t, indexes=idx)
        before = _native.launch_count()
        alone[name] = m.compute()
        launches[name] = _native.launch_count() - before
    groups = _native.retrieval_sort(idx, p, t)
    before = _native.launch_count()
    _native.retrieval_evaluate(groups, _native.RET_AP)
    per_eval = _native.launch_count() - before
    sort_launches = launches["map"] - per_eval
    assert sort_launches > per_eval
    coll = MetricCollection({"map": RetrievalMAP(), "mrr": RetrievalMRR(), "p10": RetrievalPrecision(top_k=10)}).to(DEV)
    coll.update(p, t, indexes=idx)
    before = _native.launch_count()
    out = coll.compute()
    assert _native.launch_count() - before == sort_launches + 3 * per_eval
    for name in alone:
        assert torch.equal(out[name], alone[name])


def test_state_dict_reset_and_merge_state():
    from metrics_b200.retrieval import RetrievalRecall

    g = torch.Generator().manual_seed(7)
    idx = torch.randint(0, 50, (2000,), generator=g).to(DEV)
    p = torch.rand(2000, generator=g).to(DEV)
    t = (torch.rand(2000, generator=g) < 0.3).long().to(DEV)
    a, b, whole = (RetrievalRecall(top_k=5).to(DEV) for _ in range(3))
    a.update(p[:1000], t[:1000], indexes=idx[:1000])
    b.update(p[1000:], t[1000:], indexes=idx[1000:])
    whole.update(p, t, indexes=idx)
    a.merge_state(b)
    assert torch.equal(a.compute(), whole.compute())
    c = RetrievalRecall(top_k=5).to(DEV)
    c.persistent(True)
    whole.persistent(True)
    c.load_state_dict(whole.state_dict())
    assert torch.equal(c.compute(), whole.compute())
    c.reset()
    assert c.indexes == [] and c._group_cache == {}
    c.update(p[:10], t[:10], indexes=idx[:10])
    ref = RetrievalRecall(top_k=5).to(DEV)
    ref.update(p[:10], t[:10], indexes=idx[:10])
    assert torch.equal(c.compute(), ref.compute())


def test_r_precision_float_target_raises_at_compute():
    from metrics_b200.retrieval import RetrievalRPrecision

    m = RetrievalRPrecision().to(DEV)
    m.update(torch.rand(4, device=DEV), torch.tensor([0., 1., 0., 1.], device=DEV), indexes=torch.zeros(4, dtype=torch.long, device=DEV))
    with pytest.raises(TypeError, match="only integer tensors"):
        m.compute()
