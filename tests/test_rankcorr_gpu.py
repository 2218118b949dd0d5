"""GPU: SpearmanCorrCoef / KendallRankCorrCoef (kernel K17) against the reference's goldens and against the float64 oracle
at sizes and tie structures the goldens cannot reach: 10^6 and 2^24 + 77 rows, eight outputs, constant columns and tie
groups longer than a tile, NaN rows among ties, tau-b where the reference's int64 denominator overflows, float16 past
65 504 rows; determinism, state round trips and a MetricCollection holding both metrics."""
import numpy as np
import pytest
import torch

from oracle import rank_corr as orc
from tests import rankcorr_cases as rcc

pytestmark = pytest.mark.gpu
DEV = "cuda"
TILE = 2048  # rows per tie-pass tile; the radix sort's tile is 8192


def _data(n, d, seed, ties=0, nan=0.0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, d, generator=g, dtype=torch.float64)
    y = 0.6 * x + 0.8 * torch.randn(n, d, generator=g, dtype=torch.float64)
    if ties:
        x, y = (x * ties / 4).round().clamp(-ties // 2, ties // 2), (y * ties / 4).round().clamp(-ties // 2, ties // 2)
    if nan:
        x[torch.rand(n, d, generator=g) < nan] = float("nan")
        y[torch.rand(n, d, generator=g) < nan] = float("nan")
    return x.to(dtype), y.to(dtype)


def _kendall(p, t, variant="b", alternative="two-sided"):
    from metrics_b200.functional.regression import kendall_rank_corrcoef

    tau, pv = kendall_rank_corrcoef(p.to(DEV), t.to(DEV), variant=variant, t_test=True, alternative=alternative)
    return np.atleast_1d(tau.double().cpu().numpy()), np.atleast_1d(pv.double().cpu().numpy())


def _check_kendall(p, t, variants=("a", "b", "c"), alternative="two-sided"):
    pn, tn = p.double().numpy() if p.is_floating_point() else p.numpy(), t.double().numpy() if t.is_floating_point() else t.numpy()
    for v in variants:
        tau, pv = _kendall(p, t, v, alternative)
        want_tau, want_p = orc.kendall(pn, tn, v, alternative)
        dt = "float64" if (v == "c" and p.dtype == torch.float64) else "float32"
        assert rcc.ulp_close(tau, want_tau, dt, 1), (v, tau, want_tau)
        assert rcc.ulp_close(pv, want_p, "float32", 1) or np.allclose(pv, want_p, rtol=0, atol=2 ** -40, equal_nan=True), (v, pv, want_p)


def _check_spearman(p, t):
    from metrics_b200.functional.regression import spearman_corrcoef

    got = spearman_corrcoef(p.to(DEV), t.to(DEV))
    assert got.dtype == p.dtype
    want = orc.spearman(p.double().numpy(), t.double().numpy())
    dt = str(p.dtype).replace("torch.", "")
    assert rcc.ulp_close(got.double().cpu().numpy(), want, dt, 1), (got, want)


def test_every_golden_through_classes_and_functionals():
    from metrics_b200.functional.regression import kendall_rank_corrcoef, spearman_corrcoef
    from metrics_b200.regression import KendallRankCorrCoef, SpearmanCorrCoef

    golden = rcc.load()
    for key, meta in rcc.cases(golden):
        bs = rcc.batches(golden, key, meta, DEV)
        kw = meta["kwargs"]
        num_outputs = max(meta["d"], 1)
        m = SpearmanCorrCoef(num_outputs=num_outputs) if meta["metric"] == "spearman" else KendallRankCorrCoef(num_outputs=num_outputs, **kw)
        m = m.to(DEV)
        for p, t in bs:
            m.update(p, t)
        p, t = torch.cat([b[0] for b in bs]), torch.cat([b[1] for b in bs])
        fres = spearman_corrcoef(p, t) if meta["metric"] == "spearman" else kendall_rank_corrcoef(p, t, **kw)
        for name, res in (("compute", m.compute()), ("functional", fres)):
            pv = None
            if isinstance(res, tuple):
                res, pv = res
            dt = meta[f"{name}_dtype"]
            assert str(res.dtype) == f"torch.{dt}", (key, name, res.dtype)
            want = golden[f"{key}/{name}"]
            assert res.shape == want.shape, (key, name)
            got = res.double().cpu().numpy()
            if meta["metric"] == "spearman":
                if not rcc.several_nans_per_column(meta):
                    assert rcc.ulp_close(got, want, dt, rcc.spearman_ulps(dt)), (key, name, got, want)
            elif not rcc.half_overflow(meta):
                assert rcc.ulp_close(got, want, dt, 3 if dt in ("float16", "bfloat16") else 2), (key, name, got, want)
            if pv is not None:
                assert pv.dtype == torch.float32
                gp = np.atleast_1d(golden[f"{key}/{name}_p"])
                pn = np.atleast_1d(pv.double().cpu().numpy())
                pc = p.reshape(p.shape[0], -1).double().cpu().numpy()
                tc = t.reshape(t.shape[0], -1).double().cpu().numpy()
                keep = np.array([not orc.total_pairs_tied(orc.kendall_stats(pc[:, c], tc[:, c])) for c in range(len(gp))])
                assert np.allclose(pn[keep], gp[keep], rtol=2 ** -22, atol=2 ** -26, equal_nan=True), (key, name, pn, gp)


def test_constant_column_longer_than_a_tile():
    n = 5 * 8192 + 3
    p, t = _data(n, 2, 1)
    p[:, 0] = 2.5
    _check_spearman(p, t)
    _check_kendall(p, t)
    tau, pv = _kendall(p, t)
    assert np.isnan(tau[0]) and np.isnan(pv[0])  # every pair tied in preds: tau-b is 0/0, Var(S) is 0


def test_tie_groups_crossing_tile_and_sort_tile_edges():
    # group lengths chosen so that boundaries fall just before, on and after multiples of 2048 and 8192
    lengths = [TILE - 1, 2, TILE + 1, 3 * TILE, 8192 - 5, 11, 8192 + 7, 1, 1, 4 * 8192 + 13]
    x = torch.cat([torch.full((k,), float(i)) for i, k in enumerate(lengths)])
    g = torch.Generator().manual_seed(3)
    x = x[torch.randperm(len(x), generator=g)]
    y = (x + torch.randint(0, 3, x.shape, generator=g)).float()
    _check_spearman(x, y)
    _check_kendall(x, y)


@pytest.mark.parametrize("ties", [0, 5])
def test_one_million_rows(ties):
    p, t = _data(10 ** 6, 1, 4, ties=ties)
    _check_spearman(p[:, 0], t[:, 0])
    _check_kendall(p[:, 0], t[:, 0], variants=("b",))


def test_eight_outputs_with_nans_and_ties():
    p, t = _data(100_003, 8, 5, ties=5, nan=0.02)
    p[:, 3] = torch.randn(100_003, generator=torch.Generator().manual_seed(9), dtype=torch.float64).float()
    _check_spearman(p, t)
    _check_kendall(p, t)


def test_two_pow_24_plus_77_rows():
    n = (1 << 24) + 77
    p, t = _data(n, 1, 6)
    _check_spearman(p[:, 0], t[:, 0])
    p, t = _data(n, 1, 7, ties=5)
    _check_kendall(p[:, 0], t[:, 0], variants=("b",))


def test_tau_b_past_the_reference_int64_overflow():
    n = 100_000
    p, t = _data(n, 1, 8)
    tau, _ = _kendall(p[:, 0], t[:, 0], "b")
    want, _ = orc.kendall(p[:, 0].double().numpy(), t[:, 0].double().numpy(), "b")
    assert rcc.ulp_close(tau, want, "float32", 1)
    # the reference's denominator, (n(n-1)/2 - ties)^2 in int64, wraps around at this size
    total = torch.tensor(n * (n - 1) // 2)
    assert float(total * total) != float(n * (n - 1) // 2) ** 2
    assert abs(tau[0]) > 0.3


def test_float16_spearman_past_65504_rows():
    p, t = _data(70_001, 1, 10, dtype=torch.float16)
    p, t = p[:, 0], t[:, 0]
    assert torch.isinf(torch.arange(1, 70_002, dtype=torch.float16)).any()  # the reference's half-precision ranks overflow
    _check_spearman(p, t)


def test_nan_rows_mixed_with_ties():
    p, t = _data(50_000, 1, 11, ties=5, nan=0.05)
    for alt in ("two-sided", "less", "greater"):
        _check_kendall(p[:, 0], t[:, 0], alternative=alt)
    _check_spearman(p[:, 0], t[:, 0])


def test_integer_and_mixed_dtypes():
    p, t = _data(30_000, 2, 12, ties=9)
    _check_kendall(p.long(), t.int())
    _check_kendall(p.short(), t.double())
    _check_kendall(p.bool(), t)


def test_two_runs_are_bit_identical():
    from metrics_b200.functional.regression import kendall_rank_corrcoef, spearman_corrcoef

    p, t = _data(10 ** 6, 3, 13, ties=7, nan=0.01)
    p, t = p.to(DEV), t.to(DEV)
    a = [spearman_corrcoef(p, t), *kendall_rank_corrcoef(p, t, t_test=True)]
    b = [spearman_corrcoef(p, t), *kendall_rank_corrcoef(p, t, t_test=True)]
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_state_dict_round_trip_and_collection():
    from metrics_b200 import MetricCollection
    from metrics_b200.regression import KendallRankCorrCoef, SpearmanCorrCoef

    p, t = _data(20_000, 1, 14, ties=11)
    p, t = p[:, 0].to(DEV), t[:, 0].to(DEV)
    coll = MetricCollection({"rho": SpearmanCorrCoef(), "tau": KendallRankCorrCoef(variant="c")}).to(DEV)
    coll.update(p[:12_000], t[:12_000])
    coll.update(p[12_000:], t[12_000:])
    res = coll.compute()
    want_rho = orc.spearman(p.double().cpu().numpy(), t.double().cpu().numpy())
    want_tau, _ = orc.kendall(p.double().cpu().numpy(), t.double().cpu().numpy(), "c")
    assert rcc.ulp_close(res["rho"].cpu().numpy(), want_rho, "float32", 1)
    assert rcc.ulp_close(res["tau"].cpu().numpy(), want_tau, "float32", 1)

    for cls, kw in ((SpearmanCorrCoef, {}), (KendallRankCorrCoef, {"t_test": True})):
        m = cls(**kw).to(DEV)
        m.persistent(True)
        m.update(p, t)
        m2 = cls(**kw).to(DEV)
        m2.persistent(True)
        m2.load_state_dict(m.state_dict())
        x, y = m.compute(), m2.compute()
        x, y = (x if isinstance(x, tuple) else (x,)), (y if isinstance(y, tuple) else (y,))
        assert all(torch.equal(u, v) for u, v in zip(x, y))
