"""GPU: kernel K9 (`mb200_regression_sums`) against the exact oracle of oracle/regression.py on every dtype, launch path,
alignment and size edge of the kernel.

For MSE, MAE, MAPE, SMAPE, WMAPE, R2 and explained variance the kernel's per-element terms are IEEE-exact operations on
the upcast inputs, and `terms32` is bit-identical to them (tests/test_tweedie_host.py pins that on the CPU).  What is left
between the kernel and the oracle is the order of the float64 additions, bounded by

    |kernel - oracle| <= (L_kernel + 64) * 2^-52 * sum |term|

per output, where L_kernel is the longest chain of additions behind one output (per-thread serial sum + CTA fold + ordered
sum over the CTA partials, restated from the launch code in `chain_length`) and 64 covers numpy's pairwise sum of the oracle
terms.  The inputs keep every |term| above 0.02 while that bound stays below 1e-4, so one element lost, counted twice or
read from the wrong place fails at every size tested.  The transcendental ops are checked against a higher-precision
evaluation under an error bound derived from the CUDA Math API's documented maximum ulp errors (`_transcendental_bound`).
"""
import numpy as np
import pytest
import torch

from metrics_b200 import _native
from oracle import regression as orr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [torch.float32, torch.float64, torch.float16, torch.bfloat16]
EXACT_OPS = [_native.REG_MSE, _native.REG_MAE, _native.REG_MAPE, _native.REG_SMAPE, _native.REG_WMAPE, _native.REG_R2,
             _native.REG_EXPVAR]
EPS = 1.17e-06  # the MAPE / SMAPE epsilon of the functionals
MAX_CTAS = 296  # regression.cu: partial rows the scratch holds


def np_of(x: torch.Tensor) -> np.ndarray:
    """numpy copy holding the same values: bfloat16 widened to float32 (exact), the other dtypes as they are."""
    x = x.detach().cpu()
    return x.float().numpy() if x.dtype == torch.bfloat16 else x.numpy()


def kvec(dtype) -> int:
    return 16 // torch.empty((), dtype=dtype).element_size()


def chain_length(n: int, d: int) -> int:
    """Longest chain of float64 additions behind one output (launch geometry of `mb200_regression_sums`)."""
    if n == 0:
        return 0
    if d == 1:  # flat kernel: 512 threads, fp64 shuffle (5) + 16 warp sums, up to 296 CTAs of 512 * 8 elements
        g = min(MAX_CTAS, -(-n // 4096))
        return -(-n // (g * 512)) + 8 + 5 + 16 + g
    cols = min(d, 256)
    rows = 256 // cols
    tiles = -(-d // cols)
    gx = min(max(1, -(-n // (rows * 8))), max(1, MAX_CTAS // tiles))
    return -(-n // (gx * rows)) + rows + gx


def make_pair(n: int, dtype, seed: int, extra: int = 1):
    """preds / target buffers of n + extra elements with |preds - target| in [0.4, 1.5] after rounding to `dtype` and
    |target| <~ 10: every exact-op term is at least ~0.02."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    m = n + extra
    t = torch.randn(m, generator=g, device=DEV) * 2
    sign = torch.where(torch.rand(m, generator=g, device=DEV) < 0.5, -1.0, 1.0)
    p = t + sign * (torch.rand(m, generator=g, device=DEV) + 0.5)
    return p.to(dtype), t.to(dtype)


def assert_sums(got: torch.Tensor, terms: np.ndarray, n: int, d: int, msg: str) -> None:
    """`got` [K, d] from the kernel against the oracle terms [K, n, d] under the reassociation bound above."""
    t64 = np.ascontiguousarray(np.moveaxis(terms.astype(np.float64).reshape(terms.shape[0], n, d), 1, -1))
    want, mag = t64.sum(-1), np.abs(t64).sum(-1)  # along a contiguous axis: numpy's pairwise summation
    got = got.cpu().numpy()
    assert got.shape == want.shape, msg
    bound = (chain_length(n, d) + 64) * 2.0**-52 * mag
    err = np.abs(got - want)
    bad = ~(err <= bound)
    assert not bad.any(), f"{msg}: |err| {err[bad][:4]} > bound {bound[bad][:4]} (sums {got[bad][:4]} vs {want[bad][:4]})"


def census(p: np.ndarray, t: np.ndarray) -> np.ndarray:
    """Tweedie's out-of-domain counts (#p <= 0, #t < 0, #t == 0) per column of [n, d] inputs."""
    return np.stack([(p <= 0).sum(0), (t < 0).sum(0), (t == 0).sum(0)]).astype(np.float64)


def check_all_ops(p: torch.Tensor, t: torch.Tensor, d: int, msg: str) -> None:
    n = p.numel() // d
    pn, tn = np_of(p), np_of(t)
    for op in EXACT_OPS:
        got = _native.regression_sums(p, t, op, d, 0.0, EPS)
        assert_sums(got, orr.terms32(op, pn.reshape(n, d), tn.reshape(n, d), eps=EPS), n, d, f"{msg} op {op}")
    got = _native.regression_sums(p, t, _native.REG_TWEEDIE, d, 1.5)
    np.testing.assert_array_equal(got[1:].cpu().numpy(), census(pn.reshape(n, d), tn.reshape(n, d)), err_msg=f"{msg} census")


# ---- flat kernel (d == 1) ----------------------------------------------------------------------------------------------
def flat_sizes(dtype):
    k = kvec(dtype)
    return [0, 1, k - 1, k, k + 1, 2 * k * 512 + 1, MAX_CTAS * 4096 - 1, MAX_CTAS * 4096 + 1, 2**24 + 3]


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_flat_kernel_every_size_and_alignment(dtype):
    """Vector body, the tail after it (n % kVec != 0), the scalar path of a view at a one-element offset (either input or
    both), the grid cap of 296 CTAs, and the MSE / MAE / generic / Tweedie instantiations."""
    for n in flat_sizes(dtype):
        P, T = make_pair(n, dtype, seed=n)
        for a, b in ((0, 0), (1, 0), (0, 1), (1, 1)):
            check_all_ops(P[a:a + n], T[b:b + n], 1, f"{dtype} n={n} offsets=({a},{b})")


# ---- partial kernel (d > 1) --------------------------------------------------------------------------------------------
def partial_sizes(d):
    cols = min(d, 256)
    rows = 256 // cols
    cap = max(1, MAX_CTAS // -(-d // cols))
    large = rows * 8 * cap + rows + 1  # the grid reaches its cap of 296 / col_tiles CTAs, each thread loops ~8 times
    return sorted({0, 1, max(0, 256 // d - 1), 256 // d + 1, large})


@pytest.mark.parametrize("d", [2, 3, 7, 8, 255, 256, 257, 1000, 4097])
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_partial_kernel_every_width(dtype, d):
    for n in partial_sizes(d):
        P, T = make_pair(n * d, dtype, seed=7 * d + n)
        check_all_ops(P[:n * d].reshape(n, d), T[:n * d].reshape(n, d), d, f"{dtype} d={d} n={n}")
        check_all_ops(P[1:].reshape(n, d), T[1:].reshape(n, d), d, f"{dtype} d={d} n={n} offset 1")


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_partial_kernel_more_column_tiles_than_ctas(dtype):
    """d = 76 801: 301 column tiles of 256 > 296, so the grid falls back to one CTA per column tile."""
    d = 76_801
    assert 296 * 4 * d * 8 < torch.cuda.mem_get_info()[0] // 4  # the scratch, 296 * K * d doubles, fits easily
    for n in (1, 3):
        P, T = make_pair(n * d, dtype, seed=n)
        check_all_ops(P[:n * d].reshape(n, d), T[:n * d].reshape(n, d), d, f"{dtype} d={d} n={n}")


# ---- Tweedie census ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("d", [1, 3])
def test_tweedie_census_counts_exactly(dtype, d):
    """Known numbers of p <= 0, t < 0 and t == 0 — including -0.0 (it is <= 0 and == 0, not < 0) and NaN (in none) —
    placed in the vector body, in the tail and at the start of a view at a one-element offset."""
    n = (3 * 4096 + 5) * d
    p = torch.full((n + 1,), 1.5, dtype=torch.float64)
    t = torch.full((n + 1,), 2.0, dtype=torch.float64)
    # (index, p, t): counted as (p <= 0, t < 0, t == 0)
    body = 37
    placed = [(body, 0.0, -1.0), (body + 1, -0.0, -0.0), (body + 2, float("nan"), 0.0), (body + 3, -2.0, float("nan")),
              (body + 4, float("-inf"), float("-inf")), (n - 2, float("nan"), float("nan")), (n - 1, -1e-3, 0.0),
              (1, -3.0, -0.0)]
    for i, pv, tv in placed:
        p[i], t[i] = pv, tv
    p, t = p.to(dtype).to(DEV), t.to(dtype).to(DEV)
    # by construction: 6 elements with p <= 0, 2 with t < 0, 4 with t == 0, all inside both the view at offset 0 (the
    # last one, n - 1, in the tail after the vector loop) and the view at offset 1 (index 1 is its first element)
    for a in (0, 1):
        pv, tv = p[a:a + n], t[a:a + n]
        want = census(np_of(pv).reshape(-1, d), np_of(tv).reshape(-1, d))
        assert want.sum(1).tolist() == [6, 2, 4]
        got = _native.regression_sums(pv, tv, _native.REG_TWEEDIE, d, 1.5)[1:].cpu().numpy()
        np.testing.assert_array_equal(got, want, err_msg=f"offset {a}")


# ---- determinism and layout ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_two_calls_are_bitwise_equal_for_every_instantiation(dtype):
    P, T = make_pair(3 * (1 << 20) + 3, dtype, seed=11, extra=0)
    Pp, Tp = P.abs() + 0.5, T.abs() + 0.25  # Tweedie on its domain
    for d in (1, 3):
        for op, param, (p, t) in ((_native.REG_MSE, 0.0, (P, T)), (_native.REG_MAE, 0.0, (P, T)), (_native.REG_R2, 0.0, (P, T)),
                                  (_native.REG_TWEEDIE, 1.5, (Pp, Tp))):
            a = _native.regression_sums(p, t, op, d, param, EPS)
            b = _native.regression_sums(p, t, op, d, param, EPS)
            assert torch.equal(a, b), f"d={d} op {op}"


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_non_contiguous_inputs_equal_their_contiguous_copies(dtype):
    P, T = make_pair(2 * 5 * 4099, dtype, seed=5, extra=0)
    views = [(P[::2], T[::2], 1), (P.reshape(5, -1).t(), T.reshape(5, -1).t(), 5), (P.reshape(-1, 10)[:, ::2], T.reshape(-1, 10)[:, 1::2], 5)]
    for p, t, d in views:
        assert not p.is_contiguous()
        for op in (_native.REG_MSE, _native.REG_R2, _native.REG_EXPVAR):
            got = _native.regression_sums(p, t, op, d, 0.0, EPS)
            assert torch.equal(got, _native.regression_sums(p.contiguous(), t.contiguous(), op, d, 0.0, EPS)), f"op {op} d={d}"


# ---- half-precision results of the public functionals --------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=str)
def test_half_precision_functionals_are_the_oracle_rounded(dtype):
    """Terms in float32 from the upcast inputs, sums in float64, rounded to the input dtype once before the reference's
    epilogue (DESIGN, K9): each result is within 1 ulp of the same epilogue run on the oracle's sums rounded the same way."""
    import metrics_b200.functional.regression as F
    from metrics_b200.functional.regression import metrics as M

    P, T = make_pair(1000, dtype, seed=3, extra=0)
    p2, t2 = P.reshape(200, 5), T.reshape(200, 5)
    pn, tn = np_of(P), np_of(T)
    eps = torch.finfo(dtype).eps

    def rounded(op, p, t, d=1):
        return torch.from_numpy(orr.sums(op, p, t, d, eps=EPS)).to(dtype)

    cases = {
        "mse": (F.mean_squared_error(P, T), M._mean_squared_error_compute(rounded(0, pn, tn)[0, 0], 1000)),
        "mae": (F.mean_absolute_error(P, T), M._mean_absolute_error_compute(rounded(1, pn, tn)[0, 0], 1000)),
        "mape": (F.mean_absolute_percentage_error(P, T), rounded(2, pn, tn)[0, 0] / 1000),
        "smape": (F.symmetric_mean_absolute_percentage_error(P, T), 2 * rounded(3, pn, tn)[0, 0] / 1000),
        "wmape": (F.weighted_mean_absolute_percentage_error(P, T), M._weighted_mean_absolute_percentage_error_compute(*rounded(4, pn, tn)[:, 0])),
        "r2": (F.r2_score(p2, t2, multioutput="raw_values"), M._r2_score_compute(*rounded(8, np_of(p2), np_of(t2), 5), 200, multioutput="raw_values")),
        "ev": (F.explained_variance(p2, t2, multioutput="raw_values"), M._explained_variance_compute(200, *rounded(9, np_of(p2), np_of(t2), 5), "raw_values")),
    }
    for name, (got, want) in cases.items():
        assert got.dtype == dtype, name
        got, want = got.double().cpu(), want.double()
        tol = eps * torch.exp2(torch.floor(torch.log2(want.abs())))  # 1 ulp of `want` in `dtype`
        assert torch.all((got - want).abs() <= tol), f"{name}: {got} vs {want}"


# ---- more than 2^31 elements ---------------------------------------------------------------------------------------------
def test_more_than_2_pow_31_elements():
    n = 2**31 + 5
    if torch.cuda.mem_get_info()[0] < 12 * 2**30:
        pytest.skip("needs 12 GB of free device memory")
    ones = torch.ones(n, dtype=torch.float16, device=DEV)
    zeros = torch.zeros(n, dtype=torch.float16, device=DEV)
    try:
        for op in (_native.REG_MSE, _native.REG_MAE):
            assert _native.regression_sums(ones, zeros, op).item() == float(n), f"op {op}"
    finally:
        del ones, zeros
        torch.cuda.empty_cache()


# ---- transcendental ops ----------------------------------------------------------------------------------------------
# Maximum errors in ulp, CUDA Math API (CUDA C++ Programming Guide, "Mathematical Functions"):
#   float:  logf 1, log1pf 1, expf 2, powf 4;   double: log 1, log1p 1, exp 1, pow 2.
# One ulp of a result is at most 2u of its magnitude (u = 2^-24 for float, 2^-53 for double terms).  First-order
# propagation through each formula gives err_i <= c * u * S_i with the op's S_i below; every bound here uses twice the
# derived constant c, which covers the second-order terms.
def _transcendental_bound(op, param, p, t, d, f64):
    """Per-element error bound of the kernel's terms (see above); p, t, d in longdouble."""
    ld = np.longdouble
    u = ld(2.0**-53) if f64 else ld(2.0**-24)
    if op == _native.REG_MSLE:  # l = log1p(p) - log1p(t): err(l) <= 2u(|Lp|+|Lt|) + u|l|; err(l*l) <= 2|l| err(l) + u l^2
        lp, lt = np.log1p(p), np.log1p(t)
        l = lp - lt
        return 2 * 4 * u * (np.abs(l) * (np.abs(lp) + np.abs(lt)) + l * l)
    if op == _native.REG_LOGCOSH:  # two exps (2 ulp each) + add: relative 5u; log: absolute 5u + 1 ulp of the result
        v = np.log((np.exp(d) + np.exp(-d)) / 2)
        return 2 * 5 * u * (1 + np.abs(v))
    if op == _native.REG_MINKOWSKI:  # pow: 4 ulp
        return 2 * 8 * u * np.abs(d) ** ld(param)
    # Tweedie deviance
    if param == 1:  # log(t/p): absolute u + 2u|L|; t * L, + p, - t: one rounding each
        L = np.where(t == 0, 0, np.log(np.where(t == 0, 1, t / p)))
        return 2 * 3 * u * 2 * (np.abs(t) * (1 + np.abs(L)) + np.abs(t * L) + np.abs(p) + np.abs(t))
    if param == 2:
        L = np.log(p / t)
        return 2 * 3 * u * 2 * (1 + np.abs(L) + np.abs(t / p) + 1)
    a, b = ld(1 - param), ld(2 - param)  # three pow / (mul) / div pieces: <= 10u each, two adds
    A = np.maximum(t, 0) ** b / (a * b)
    B = t * p**a / a
    C = p**b / b
    return 2 * 12 * u * 2 * (np.abs(A) + np.abs(B) + np.abs(C))


def _exact_terms(op, param, p, t, d):
    ld = np.longdouble
    if op == _native.REG_MSLE:
        return (np.log1p(p) - np.log1p(t)) ** 2
    if op == _native.REG_LOGCOSH:
        return np.log((np.exp(d) + np.exp(-d)) / 2)
    if op == _native.REG_MINKOWSKI:
        return np.abs(d) ** ld(param)
    if param == 1:
        return 2 * (np.where(t == 0, 0, t * np.log(np.where(t == 0, 1, t / p))) + p - t)
    if param == 2:
        return 2 * (np.log(p / t) + t / p - 1)
    a, b = ld(1 - param), ld(2 - param)
    return 2 * (np.maximum(t, 0) ** b / (a * b) - t * p**a / a + p**b / b)


TRANSCENDENTAL = [(_native.REG_MSLE, 0.0), (_native.REG_LOGCOSH, 0.0), (_native.REG_MINKOWSKI, 1.5), (_native.REG_MINKOWSKI, 3.0),
                  (_native.REG_TWEEDIE, 1.0), (_native.REG_TWEEDIE, 1.5), (_native.REG_TWEEDIE, 2.0), (_native.REG_TWEEDIE, 3.0),
                  (_native.REG_TWEEDIE, -1.0)]


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("op,param", TRANSCENDENTAL, ids=lambda x: str(x))
def test_transcendental_ops_within_the_derived_ulp_bound(dtype, op, param):
    g = torch.Generator(device=DEV).manual_seed(op * 10 + int(param * 2) + 5)
    f64 = dtype == torch.float64
    for n, d in ((1, 1), (1000, 1), (65537, 1), (4001, 3)):
        m = n * d
        if op == _native.REG_LOGCOSH or op == _native.REG_MINKOWSKI:
            p = torch.randn(m, generator=g, device=DEV, dtype=torch.float64) * 3
            t = torch.randn(m, generator=g, device=DEV, dtype=torch.float64) * 3
        else:  # MSLE and Tweedie: positive preds, positive targets (some exactly 0 where the power allows it)
            p = torch.rand(m, generator=g, device=DEV, dtype=torch.float64) * 4 + 0.25
            t = p * torch.exp(torch.randn(m, generator=g, device=DEV, dtype=torch.float64) * 0.5)
            if op == _native.REG_TWEEDIE and 1 <= param < 2:
                t[::7] = 0
        p, t = p.to(dtype), t.to(dtype)
        got = _native.regression_sums(p, t, op, d, param).cpu().numpy()[0]
        pn, tn = np_of(p).reshape(n, d), np_of(t).reshape(n, d)
        # the kernel's own difference (an IEEE-exact operation) feeds LogCosh and Minkowski
        f = np.float64 if f64 else np.float32
        dn = (pn.astype(f) - tn.astype(f)).astype(np.longdouble)
        pl, tl = pn.astype(np.longdouble), tn.astype(np.longdouble)
        with np.errstate(divide="ignore", invalid="ignore"):
            exact = _exact_terms(op, param, pl, tl, dn)
            bound = _transcendental_bound(op, param, pl, tl, dn, f64)
        want = exact.sum(0)
        sum_bound = bound.sum(0) + (chain_length(n, d) + 64) * 2.0**-52 * np.abs(exact).sum(0)
        err = np.abs(got.astype(np.longdouble) - want)
        assert np.all(err <= sum_bound), f"{dtype} op {op} param {param} n={n} d={d}: err {err} > {sum_bound}"


# ---- the reference's goldens on mixed dtypes, N-d inputs, num_outputs not the row width ----------------------------------
def test_replay_reference_goldens_on_the_kernel():
    import os

    from tests.conftest import GOLDEN_DIR
    from tests.regression_dtype_cases import replay

    g = np.load(os.path.join(GOLDEN_DIR, "regression_dtypes.npz"), allow_pickle=False)
    assert replay(g, DEV) == int(g["n_cases"])


def test_same_dtype_call_adds_no_cast_and_two_launches():
    p, t = make_pair(1 << 16, torch.float32, seed=1, extra=0)
    before = _native.launch_count()
    _native.regression_sums(p, t, _native.REG_MSE)
    assert _native.launch_count() - before == 2
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU]) as prof:
        _native.regression_sums(p, t, _native.REG_MSE)
    assert "aten::_to_copy" not in {e.key for e in prof.key_averages()}


def test_num_outputs_must_divide_the_element_count():
    with pytest.raises(ValueError, match="num_outputs=3"):
        _native.regression_sums(torch.zeros(10, 4, device=DEV), torch.zeros(10, 4, device=DEV), _native.REG_MSE, 3)
