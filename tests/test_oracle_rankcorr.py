"""CPU: the float64 rank-correlation oracle (oracle/rank_corr.py) against the reference's goldens and against scipy, and its
O(n log n) inversion count against a brute-force count."""
import math

import numpy as np
import pytest
import scipy.stats as ss
import torch

from oracle import rank_corr as orc
from tests import rankcorr_cases as rcc


def _concat(golden, key, meta):
    bs = rcc.batches(golden, key, meta)
    p, t = torch.cat([b[0] for b in bs]), torch.cat([b[1] for b in bs])
    return p.double().numpy() if p.is_floating_point() else p.numpy(), t.double().numpy() if t.is_floating_point() else t.numpy()


def test_oracle_matches_every_golden():
    golden = rcc.load()
    checked = 0
    for key, meta in rcc.cases(golden):
        p, t = _concat(golden, key, meta)
        kw = meta["kwargs"]
        if meta["metric"] == "spearman":
            if rcc.several_nans_per_column(meta):
                continue
            want = golden[f"{key}/functional"]
            dt = meta["functional_dtype"]
            assert rcc.ulp_close(orc.spearman(p, t).astype(np.float64), want, dt, rcc.spearman_ulps(dt)), key
        else:
            alt = kw.get("alternative", "two-sided") if kw.get("t_test") else None
            tau, pv = orc.kendall(p, t, kw.get("variant", "b"), alt)
            want = np.atleast_1d(golden[f"{key}/functional"])
            dt = meta["functional_dtype"]
            if rcc.half_overflow(meta):
                pass
            elif dt in ("float16", "bfloat16"):  # variant c in half precision: three half-precision roundings
                assert rcc.ulp_close(tau, want, dt, 3), key
            else:
                assert rcc.ulp_close(tau, want, "float32" if dt == "float32" else dt, 2), key
            if alt is not None:
                gp = np.atleast_1d(golden[f"{key}/functional_p"])
                tied = [orc.total_pairs_tied(orc.kendall_stats(p.reshape(len(p), -1)[:, c], t.reshape(len(t), -1)[:, c]))
                        for c in range(len(gp))]
                keep = ~np.array(tied)
                assert np.allclose(pv[keep], gp[keep], rtol=2 ** -22, atol=2 ** -26, equal_nan=True), key
        checked += 1
    assert checked >= 120


@pytest.mark.parametrize("seed", range(4))
def test_oracle_matches_scipy(seed):
    g = np.random.default_rng(seed)
    for n, levels in ((1, 0), (2, 0), (300, 0), (2000, 5), (5000, 0)):
        x = g.normal(size=n)
        y = 0.5 * x + g.normal(size=n)
        if levels:
            x, y = np.round(x * 1.2).clip(-2, 2), np.round(y).clip(-2, 2)
        if n >= 3:
            rho = ss.spearmanr(x, y)[0]
            assert math.isclose(orc.spearman(x, y, eps=0.0)[0], rho, rel_tol=1e-12, abs_tol=1e-14)
            for variant in ("b", "c"):
                want = ss.kendalltau(x, y, variant=variant)
                tau, pv = orc.kendall(x, y, variant, "two-sided")
                assert math.isclose(tau[0], want.statistic, rel_tol=1e-12, abs_tol=1e-14)
                if variant == "b" and n > 10:
                    asym = ss.kendalltau(x, y, variant="b", method="asymptotic").pvalue
                    assert math.isclose(pv[0], asym, rel_tol=1e-9, abs_tol=1e-300)


def test_inversion_count_matches_brute_force():
    g = np.random.default_rng(7)
    for n, hi in ((1, 1), (2, 2), (17, 3), (200, 5), (300, 1000), (257, 256)):
        s = g.integers(0, hi, size=n)
        brute = int(sum(int((s[i] > s[i + 1:]).sum()) for i in range(n)))
        assert orc.count_inversions(s) == brute
