"""CPU: Tweedie deviance.  (a) the host layer against goldens from the reference, kernel replaced by its stand-in;
(b) the kernel's own term function (csrc/regression_terms.cuh), compiled for the host by nvcc, element by element against
the reference — so the formulas the GPU runs are checked here even without a GPU."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests.conftest import ROOT
from tests.tweedie_cases import domain_errors, replay


def test_replay_reference_goldens(golden_tweedie, cpu_kernel_standins):
    assert replay(golden_tweedie, "cpu") == 24


def test_domain_errors_and_corners(cpu_kernel_standins):
    domain_errors("cpu")


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("reg_terms") / "reg_terms_host")
    src = os.path.join(ROOT, "metrics_b200", "csrc", "tools", "reg_terms_host.cu")
    build = subprocess.run([nvcc, "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets", "-o", exe, src],
                           capture_output=True, text=True)
    assert build.returncode == 0, build.stderr[-2000:]

    def run(op, param, eps, precision, preds, targets):
        lines = "".join(f"{p!r} {t!r}\n" for p, t in zip(preds.tolist(), targets.tolist()))
        out = subprocess.run([exe, str(op), repr(float(param)), repr(float(eps)), precision], input=lines, capture_output=True,
                             text=True, check=True).stdout
        return np.array([[float(v) for v in row.split()] for row in out.strip().splitlines()])

    return run


@pytest.mark.parametrize("precision,rtol,atol", [("f64", 1e-13, 1e-14), ("f32", 3e-6, 2e-6)])  # atol: p == t gives 0 +- rounding
def test_kernel_term_function_matches_the_reference_per_element(golden_tweedie, harness, precision, rtol, atol):
    g = golden_tweedie
    preds = g["elem/preds"]
    for power in g["powers"].tolist():
        if power == 0:
            continue  # served by the squared-error op
        targets = g[f"elem/p{power}/targets"]
        terms = harness(10, power, 0.0, precision, preds, targets)
        np.testing.assert_allclose(terms[:, 0], g[f"elem/p{power}/deviance"], rtol=rtol, atol=atol, err_msg=f"power {power}")
        np.testing.assert_array_equal(terms[:, 1], (preds <= 0).astype(float))
        np.testing.assert_array_equal(terms[:, 2], (targets < 0).astype(float))
        np.testing.assert_array_equal(terms[:, 3], (targets == 0).astype(float))
    census = harness(10, 2.0, 0.0, precision, np.array([0.0, -1.0, 2.0]), np.array([-3.0, 0.0, 1.0]))
    assert census[:, 1:].tolist() == [[1, 1, 0], [1, 0, 1], [0, 0, 0]]


def test_the_other_ops_are_untouched_by_the_shared_header(harness):
    p, t = np.array([1.5, -2.0, 0.25]), np.array([1.0, 3.0, 0.25])
    d = p - t
    np.testing.assert_allclose(harness(0, 0, 0, "f64", p, t)[:, 0], d * d)
    np.testing.assert_allclose(harness(1, 0, 0, "f64", p, t)[:, 0], np.abs(d))
    np.testing.assert_allclose(harness(2, 0, 1.17e-6, "f64", p, t)[:, 0], np.abs(d) / np.maximum(np.abs(t), 1.17e-6))
    np.testing.assert_allclose(harness(7, 3.0, 0, "f64", p, t)[:, 0], np.abs(d) ** 3)
    np.testing.assert_allclose(harness(4, 0, 0, "f64", p, t), np.stack([np.abs(d), np.abs(t)], 1))
    np.testing.assert_allclose(harness(8, 0, 0, "f64", p, t), np.stack([t * t, t, (t - p) ** 2], 1))
    np.testing.assert_allclose(harness(9, 0, 0, "f64", p, t), np.stack([t - p, (t - p) ** 2, t, t * t], 1))


def _special_pairs(dtype):
    """Every pair of special values (±0, NaN, ±inf, the extremes and subnormals of `dtype`, small integers) and random
    values over a wide range of magnitudes, as float64 arrays holding `dtype` values exactly."""
    fi = np.finfo(dtype)
    tiny_sub = float(fi.smallest_subnormal)
    specials = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, float(fi.max), -float(fi.max), float(fi.tiny), -float(fi.tiny),
                         tiny_sub, -tiny_sub, 3 * tiny_sub, float(fi.tiny) / 3, 1.0, -1.0, 2.0, 0.5, 1e-7, -3.25], dtype=dtype)
    p, t = np.meshgrid(specials, specials)
    rng = np.random.default_rng(7)
    n = 2000
    rp = (rng.standard_normal(n) * 10.0 ** rng.integers(-30, 30, n)).astype(dtype)
    rt = (rp.astype(np.float64) * (1 + rng.standard_normal(n) * 10.0 ** rng.integers(-8, 1, n))).astype(dtype)
    p = np.concatenate([p.ravel(), rp, rng.standard_normal(n).astype(dtype)])
    t = np.concatenate([t.ravel(), rt, rng.standard_normal(n).astype(dtype)])
    return p.astype(np.float64), t.astype(np.float64)


def _bitwise_equal(a, b):
    """Equal bit patterns, except that any NaN matches any NaN (the harness prints NaN without its payload)."""
    both_nan = np.isnan(a) & np.isnan(b)
    same = a.view(np.uint64) == b.view(np.uint64)
    return bool(np.all(both_nan | same)), np.flatnonzero(~(both_nan | same))


@pytest.mark.parametrize("precision,dtype", [("f32", np.float32), ("f64", np.float64)])
@pytest.mark.parametrize("op", [0, 1, 2, 3, 4, 8, 9])
def test_oracle_terms_are_bitwise_the_kernel_term_function(harness, precision, dtype, op):
    """oracle/regression.py `terms32` against the kernel's own `reg_terms` for the ops made only of IEEE-exact operations:
    bit for bit, on special, extreme and random values, so that the GPU suite can hold the kernel to exact sums."""
    from oracle import regression as orr

    p, t = _special_pairs(dtype)
    for eps in ((1.17e-06, 0.0) if op in (2, 3) else (0.0,)):
        got = harness(op, 0.0, eps, precision, p, t).T  # [K, n], float64 holding the kernel's term values exactly
        want = orr.terms32(op, p.astype(dtype), t.astype(dtype), eps=eps).astype(np.float64)
        assert got.shape == want.shape
        ok, bad = _bitwise_equal(got, want)
        assert ok, f"op {op} eps {eps}: first mismatches at p={p[bad[:4] % p.size]}, t={t[bad[:4] % p.size]}"


def test_oracle_terms_of_half_inputs_are_the_float32_terms_of_the_upcast_values():
    from oracle import regression as orr

    rng = np.random.default_rng(3)
    for half in (np.float16,):
        p, t = rng.standard_normal(1000).astype(half), rng.standard_normal(1000).astype(half)
        for op in (0, 3, 9):
            got = orr.terms32(op, p, t, eps=1.17e-6)
            assert got.dtype == np.float32
            np.testing.assert_array_equal(got, orr.terms32(op, p.astype(np.float32), t.astype(np.float32), eps=1.17e-6))
