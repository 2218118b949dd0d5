"""CPU: oracle/normalize.py (`normalize_logits_if_needed` restated) against goldens from the unmodified reference
(tests/golden/make_golden_normalize.py): every float dtype, 1-D sigmoid and `[N, C]` / `[N, C, d]` / `[N, C, h, w]` softmax
batches, logits and probabilities, exact 0 / -0.0 / 1 and single scores one step outside [0, 1].  `chain` must give the
reference's bits, `exact` must lie within `bound` of them, the bound must fail a softmax that drops one summand, and
`path_of` must give the literal launch paths the GPU suite (tests/test_normalize_paths_gpu.py) relies on."""
import os

import numpy as np
import pytest
import torch

from metrics_b200 import _native
from oracle import normalize as on
from tests.conftest import GOLDEN_DIR

DTYPES = {0: torch.float32, 1: torch.float16, 2: torch.bfloat16, 3: torch.float64}
F16, BF16, F32, F64 = torch.float16, torch.bfloat16, torch.float32, torch.float64


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN_DIR, "normalize.npz"), allow_pickle=False)


def sets(g):
    for i in range(int(g["n_sets"])):
        key = f"set{i}"
        code, softmax = (int(v) for v in g[f"{key}/meta"])
        dtype = DTYPES[code]
        x = torch.from_numpy(g[f"{key}/x"]).to(dtype)
        y = torch.from_numpy(g[f"{key}/y"]).to(dtype)
        yield key, "softmax" if softmax else "sigmoid", x, y, str(g[f"{key}/kind"])


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.view({8: torch.int64, 4: torch.int32, 2: torch.int16}[t.element_size()])


def test_chain_reproduces_every_golden_bit_for_bit(golden):
    kinds = set()
    for key, norm, x, y, kind in sets(golden):
        got = on.chain(x, norm)
        assert got.dtype == y.dtype and torch.equal(bits(got), bits(y)), (key, norm, x.dtype, kind)
        kinds.add((norm, x.dtype, x.ndim, kind))
    assert len(kinds) == 4 * 5 + 4 * 3 * 5  # every (normalisation, dtype, rank, kind) seen


def test_golden_votes(golden):
    """Exact 0, -0.0 and 1 are probabilities (passed through with their bits); one step outside [0, 1] makes logits."""
    for key, norm, x, y, kind in sets(golden):
        assert on.is_logits(x) == (kind in ("logits", "below", "above")), (key, kind)
        if kind in ("probs", "edges"):
            assert torch.equal(bits(y), bits(x)), key
    neg0 = torch.tensor([0.5, -0.0, 1.0])
    assert not on.is_logits(neg0) and torch.equal(bits(on.chain(neg0, "sigmoid")), bits(neg0))
    assert not on.is_logits(torch.tensor([float("nan"), 0.25]))


def test_exact_within_bound_of_every_golden(golden):
    """ATen's CPU softmax over a dim that is not the last one keeps float16 / bfloat16 intermediates (up to 1.3 ulp off
    here), so those goldens are held to 2 ulp of `exact`; every other golden to `bound`, the kernels' float32 arithmetic."""
    for key, norm, x, y, kind in sets(golden):
        if x.ndim > 2 and x.dtype in (F16, BF16):
            e = on.exact(x, norm)
            assert (np.abs(y.double().numpy() - e) <= 2 * on.ulp(e, x.dtype)).all(), (key, x.dtype, kind)
            continue
        nbad, worst = on.violations(y, x, norm)
        assert nbad == 0, (key, norm, x.dtype, kind, worst)


def test_bound_fails_a_dropped_summand_and_a_few_ulp():
    """The softmax bound is far tighter than one summand of the row sum; the sigmoid bound is a few ulp."""
    g = torch.Generator().manual_seed(5)
    for dtype in (F32, F16, BF16, F64):
        for c in (2, 33, 64, 513, 1024, 2048):
            x = (torch.randn(64, c, generator=g, dtype=F64) * 3).to(dtype)
            assert on.violations(on.chain(x, "softmax"), x, "softmax")[0] == 0, (dtype, c)
            for drop in (0, c - 1):  # a lane (C <= 32) or an iteration (C > 32) left out of the sum
                keep = torch.ones(c, dtype=torch.bool)
                keep[drop] = False
                e = torch.exp(x.double() - x.double().amax(1, keepdim=True))
                bad = (e / (e * keep).sum(1, keepdim=True)).to(dtype)
                assert on.violations(bad, x, "softmax")[0] > 0, (dtype, c, drop)
    x = torch.linspace(-20, 20, 4001, dtype=F64).to(F32)
    y = on.chain(x, "sigmoid")
    assert on.violations(y, x, "sigmoid")[0] == 0
    off = torch.nextafter(y, torch.full_like(y, 2.0))
    for _ in range(7):
        off = torch.nextafter(off, torch.full_like(off, 2.0))
    assert on.violations(off, x, "sigmoid")[0] > 1000  # 8 ulp up is outside
    b = on.bound(x, "sigmoid") / on.ulp(on.exact(x, "sigmoid"), F32)
    assert b.max() <= 6.01 and b[x.numpy() < 0].max() > 4


def test_bound_covers_the_overflow_and_subnormal_edges():
    """exp(-x) overflows float32 above 88.72 and float64 above 709.78: 1 / (1 + inf) is 0, which the bound admits; float32
    sigmoids near -103.97 are subnormal, where the floor of one subnormal step applies."""
    x32 = torch.tensor([-88.7, -88.8, -90.0, -103.9, -104.0, -200.0, float("-inf"), 17.0, 88.8, float("inf")])
    y32 = 1 / (1 + torch.exp(-x32))
    assert on.violations(y32, x32, "sigmoid")[0] == 0
    assert float(y32[2]) == 0.0 and on.exact(x32, "sigmoid")[2] > 0
    x64 = torch.tensor([-709.7, -709.8, -745.1, -745.2, -800.0, 36.0, 38.0], dtype=F64)
    assert on.violations(1 / (1 + torch.exp(-x64)), x64, "sigmoid")[0] == 0


def test_softmax_special_rows():
    """One +inf, a NaN or all -inf make the row NaN in the kernels and in `exact`; other rows keep their values."""
    x = torch.tensor([[1.0, float("inf"), 0.5], [float("nan"), 2.0, 0.0], [float("-inf")] * 3, [-1e30, 1e30, 0.0],
                      [2.0, 2.0, -2.0]])
    e = on.exact(x, "softmax")
    assert np.isnan(e[:3]).all() and not np.isnan(e[3:]).any()
    assert e[3].tolist() == [0.0, 1.0, 0.0] and e[4, 0] == e[4, 1]
    assert on.violations(on.chain(x, "softmax"), x, "softmax")[0] == 0


def test_nd_softmax_folds_rows_over_the_class_dim():
    g = torch.Generator().manual_seed(9)
    x = torch.randn(3, 5, 4, 2, generator=g, dtype=F64)
    want = torch.softmax(x, 1).numpy()
    assert np.abs(on.exact(x, "softmax") - want).max() < 1e-15
    assert on.violations(torch.softmax(x.float(), 1), x.float(), "softmax")[0] == 0


@pytest.mark.parametrize("torch_binding", [False, True])
@pytest.mark.parametrize("shape", [(), (5,)])
def test_softmax_rejects_inputs_without_a_class_dim(monkeypatch, torch_binding, shape):
    """Both bindings raise the same error for a 0-d or 1-D softmax input, before any device work."""
    monkeypatch.setattr(_native, "_TORCH_BINDING", torch_binding)
    with pytest.raises(ValueError, match=r"softmax normalisation expects an \[N, C, \.\.\.\] tensor"):
        _native.softmax_if_logits(torch.zeros(shape))


def test_path_of_literal_expectations():
    P = on.path_of
    # sigmoid
    assert P("sigmoid", F32, 32768) == dict(kernel="small", grid=1)
    assert P("sigmoid", F64, 12288) == dict(kernel="small", grid=1)
    assert P("sigmoid", F64, 12289) == dict(kernel="flag", grid=7, head=0, vectors=0, tail=12289)
    assert P("sigmoid", F32, 32769) == dict(kernel="spec", tiles=9, extra_tile=True, grid=9, tiles_per_cta=1, tail=1)
    assert P("sigmoid", F32, 32769, binding="torch") == dict(kernel="flag", grid=17, head=0, vectors=8192, tail=1)
    assert P("sigmoid", F32, 32769, offset=1) == dict(kernel="flag", grid=17, head=3, vectors=8191, tail=2)
    assert P("sigmoid", F16, 65537, offset=5) == dict(kernel="flag", grid=33, head=3, vectors=8191, tail=6)
    assert P("sigmoid", F32, 40000, binding="abi", scratch="misaligned")["kernel"] == "flag"
    assert P("sigmoid", F32, 4096 * 12 + 3) == dict(kernel="spec", tiles=13, extra_tile=True, grid=13, tiles_per_cta=1, tail=3)
    assert P("sigmoid", F16, 8192 * 12 + 7)["extra_tile"] and not P("sigmoid", F16, 8192 * 12 + 8)["extra_tile"]
    assert P("sigmoid", F32, 1 << 23) == dict(kernel="spec", tiles=2048, extra_tile=False, grid=1056, tiles_per_cta=2, tail=0)
    assert P("sigmoid", F16, (1 << 31) + 5)["tiles_per_cta"] == 249
    # softmax
    assert P("softmax", F32, 100, 1) == dict(kernel="spec", kiter=1, grid=13, rows_per_warp=1)
    for c, k in ((32, 1), (33, 2), (64, 2), (65, 4), (128, 4), (129, 8), (256, 8), (257, 16), (512, 16), (513, 32),
                 (1024, 32)):
        assert P("softmax", BF16, 8, c)["kiter"] == k, c
    assert P("softmax", F32, 3169, 7) == dict(kernel="spec", kiter=1, grid=396, rows_per_warp=2)
    assert P("softmax", F32, 3168, 7)["rows_per_warp"] == 1
    assert P("softmax", F32, 64, 1025)["kernel"] == "flag"
    assert P("softmax", F64, 64, 3)["kernel"] == "flag"
    assert P("softmax", F16, 64, 3, binding="torch")["kernel"] == "flag"
    assert P("softmax", F32, 64, 3, binding="abi", scratch="short")["kernel"] == "flag"
    assert P("softmax", F32, 9000, 5, binding="torch") == dict(kernel="flag", grid=1056, rows_per_warp=2)
    # K11
    assert P("fused", F32, 3169, 65, target_dtype=torch.int32) == dict(kernel="fused", kiter=4, load="load_label", grid=396,
                                                                       rows_per_warp=2)
    assert P("fused", F16, 10, 1)["load"] == "kI64" and P("fused", F16, 10, 1)["kiter"] == 1
