"""Oracle for logit normalisation (kernel K6, csrc/curve.cu, and the softmax half of K11, csrc/fused.cu).  TEST
INFRASTRUCTURE ONLY — see oracle/__init__.py.

Three pieces:

  * `chain(x, normalization)`: the reference's device branch (utilities/compute.py:223-229), restated as
    `torch.where(((x < 0) | (x > 1)).any(), torch.sigmoid(x) | torch.softmax(x, 1), x)`.  NaN does not vote (it compares
    false both ways) and -0.0 is not below 0.  Run on the kernel's GPU it is the arbiter for bit equality; run on the CPU it
    reproduces the reference's CPU branch whenever the batch holds no NaN (tests/golden/normalize.npz).
  * `exact(x, normalization)`: the same computation without ATen, in numpy: float64 for float32 / float16 / bfloat16 inputs,
    `np.longdouble` (64 or more significand bits) for float64 inputs.  NaN where the arithmetic makes NaN.
  * `bound(x, normalization, dtype)`: how far a correct kernel may lie from `exact`, element by element (derivation below).
    `violations` applies it.

Forward-error bounds.  `u` is the unit roundoff of the compute type (2^-24 for float32, which float16 / bfloat16 inputs are
computed in; 2^-53 for float64), `ulp_T(y)` the spacing of the output dtype T at y (the subnormal step below its normal
range), and `step_T` the subnormal step of T.

Sigmoid, `1 / (1 + exp(-x))` in the compute type.  With `e = exp(-x)` and `y = 1 / (1 + e)`, an error `d` relative in `e`
moves `1 + e` by `d * e / (1 + e) = d * (1 - y)` relative; the add and the division round once each (`u` each).  CUDA's
`expf` is within 2 ulp (`<= 4u` relative), `exp` within 1 ulp (`<= 2u`), so

    |got - y| <= y * (eps_exp * (1 - y) + 2u) + step_T          (float32, float64: eps_exp = 4u, 2u)

which is at most 6 ulp of y for float32 (ulp(y) > u * y) and at most 4 ulp where y >= 1/2, and at most 4 ulp for float64.
float16 / bfloat16 round that float32 result once more: `|got - y| <= ulp_T(y)` (half an ulp of T plus a float32 error
thousands of times smaller).  Where `exp(-x)` overflows the compute type (`-x > 88.72` in float32, `-x > 709.78` in float64)
the formula gives exactly 0 while y is below 1 / FLT_MAX (1 / DBL_MAX): there the bound also admits y itself.

Softmax over dim 1, the kernels' order (row maximum m; `e_i = exp(x_i - m)`; lane-strided partial sums of at most
ceil(C/32) terms, a 5-level butterfly; `e_i / s`):

    |got_i - y_i| <= ulp_T(y_i) + 2 y_i u (|x_i - m| + 2 + sum_j y_j (|x_j - m| + 2) + ceil(C/32) + 6) + 2 step_c

term by term: the rounding of the exp argument (`u |x_i - m|` relative in e_i), the exponential (2u), the same two errors
carried by every summand into s (weighted by y_j = e_j / s), the ceil(C/32) - 1 lane adds and 5 butterfly adds, the
division, all doubled to turn first-order relative errors into a bound; `ulp_T(y_i)` is the final rounding to T, `2 step_c`
(step of the compute type) the absolute error of an exponential that underflows into the subnormal range.  A dropped lane
or iteration removes a whole summand `e_j` from s, and changes y_i by a relative `y_j`: for the rows these tests use that is
orders of magnitude above the bound.

Where the batch holds no score outside [0, 1] the output is the input: the bound is 0.

`path_of` restates the launch dispatch of `_native`, csrc/curve.cu and csrc/fused.cu, so that each GPU case can assert
which kernels it runs before it runs them.
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch
from torch import Tensor

# significand bits, minimum normal exponent of each output dtype
_FMT = {torch.float32: (23, -126), torch.float16: (10, -14), torch.bfloat16: (7, -126), torch.float64: (52, -1022)}
_LOG_MAX = {False: 88.72, True: 709.78}  # exp(-x) overflows the compute type above these (float32, float64)
SMALL_N = 32768  # sigmoid_if_small_kernel: 1024 threads x kSmallItems
SMALL_N_F64 = 12288  # 1024 x kSmallItemsF64
TILE_VECS = 1024  # kSpecTileVecs: 16-byte vectors per speculative sigmoid tile


def _wide():
    assert np.finfo(np.longdouble).nmant >= 63, "np.longdouble has no extended precision here"
    return np.longdouble


def _to_numpy(x: Tensor) -> np.ndarray:
    x = x.detach().cpu()
    with np.errstate(invalid="ignore"):  # NaN payloads
        if x.dtype == torch.float64:
            return x.numpy().astype(_wide())
        return x.float().numpy().astype(np.float64)


def ulp(y: np.ndarray, dtype: torch.dtype) -> np.ndarray:
    """Spacing of `dtype` at |y| (the subnormal step below its normal range); NaN / inf give NaN / inf."""
    p, emin = _FMT[dtype]
    a = np.abs(y)
    _, e = np.frexp(np.where(np.isfinite(a), a, 1))
    e = np.maximum(e.astype(np.int64) - 1, emin)
    out = np.ldexp(np.ones_like(a), e - p)
    return np.where(np.isfinite(a), out, np.inf)


def step(dtype: torch.dtype) -> float:
    p, emin = _FMT[dtype]
    return math.ldexp(1.0, emin - p)


def is_logits(x: Tensor) -> bool:
    """The reference's device vote: any score below 0 or above 1; NaN never votes, -0.0 is not below 0."""
    return bool(((x < 0) | (x > 1)).any())


def chain(x: Tensor, normalization: str) -> Tensor:
    """utilities/compute.py:223-229 (the device branch), on x's device."""
    condition = ((x < 0) | (x > 1)).any()
    return torch.where(condition, torch.sigmoid(x) if normalization == "sigmoid" else torch.softmax(x, dim=1), x)


def _rows(x: Tensor) -> Tensor:
    """`[M, C]` rows of an `[N, C, ...]` tensor, class dim last."""
    return x.movedim(1, -1).reshape(-1, x.shape[1]) if x.ndim > 2 else x


def _unrows(a: np.ndarray, like: Tensor) -> np.ndarray:
    if like.ndim <= 2:
        return a
    moved = (like.shape[0], *like.shape[2:], like.shape[1])
    return np.moveaxis(a.reshape(moved), -1, 1)


def _softmax_parts(r: np.ndarray):
    with np.errstate(invalid="ignore", over="ignore", under="ignore", divide="ignore"):
        m = np.max(r, axis=1, keepdims=True)  # NaN in a row makes the row NaN, as in the kernels
        e = np.exp(r - m)
        s = e.sum(axis=1, keepdims=True)
        return m, e / s


def exact(x: Tensor, normalization: str) -> np.ndarray:
    """What the normalisation computes, in float64 (float64 inputs: np.longdouble), shaped like x."""
    a = _to_numpy(x)
    if not is_logits(x):
        return a
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        if normalization == "sigmoid":
            return 1 / (1 + np.exp(-a))
    r = _to_numpy(_rows(x))
    return _unrows(_softmax_parts(r)[1], x)


def bound(x: Tensor, normalization: str, dtype: Optional[torch.dtype] = None) -> np.ndarray:
    """Largest |got - exact| a correct kernel may produce, element by element (see the module docstring)."""
    dtype = dtype or x.dtype
    f64 = dtype == torch.float64
    a = _to_numpy(x)
    if not is_logits(x):
        return np.zeros_like(a)
    u = 2.0 ** -53 if f64 else 2.0 ** -24
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        if normalization == "sigmoid":
            y = 1 / (1 + np.exp(-a))
            if dtype in (torch.float32, torch.float64):
                eps_exp = 2 * u if f64 else 4 * u
                b = y * (eps_exp * (1 - y) + 2 * u) * (1 + 2.0 ** -20) + step(dtype)
            else:
                b = ulp(y, dtype)
            return np.where(-a > _LOG_MAX[f64], np.maximum(b, y + step(dtype)), b)
        r = _to_numpy(_rows(x))
        m, y = _softmax_parts(r)
        d = np.abs(r - m) + 2
        carried = (y * d).sum(axis=1, keepdims=True)
        c = r.shape[1]
        b = ulp(y, dtype) + 2 * y * u * (d + carried + math.ceil(c / 32) + 6) + 2 * step(torch.float64 if f64 else torch.float32)
        return _unrows(b, x)


def violations(got: Tensor, x: Tensor, normalization: str) -> tuple[int, str]:
    """(number of elements outside the bound, a description of the worst one).  NaN must be NaN exactly where `exact` is."""
    want = exact(x, normalization)
    b = bound(x, normalization, got.dtype)
    g = _to_numpy(got)
    nan_w, nan_g = np.isnan(want), np.isnan(g)
    with np.errstate(invalid="ignore"):
        err = np.where(nan_w | nan_g, 0, np.abs(g - want))
        err = np.where(np.isinf(want) & (g == want), 0, err)
    bad = (nan_w != nan_g) | (err > b)
    nbad = int(bad.sum())
    if not nbad:
        return 0, ""
    i = np.unravel_index(int(np.argmax(np.where(bad, np.where(nan_w != nan_g, np.inf, err / np.maximum(b, 1e-300)), -1))),
                         bad.shape)
    return nbad, (f"{nbad} outside the bound; worst at {tuple(int(k) for k in i)}: x={float(_to_numpy(x)[i])!r} "
                  f"got={float(g[i])!r} exact={float(want[i])!r} bound={float(b[i])!r}")


# ----------------------------------------------------------------------------------------------------------------------
# the dispatch, restated
# ----------------------------------------------------------------------------------------------------------------------
def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


def path_of(kernel: str, dtype: torch.dtype, n: int, c: int = 1, *, binding: str = "ctypes", offset: int = 0,
            scratch: str = "owned", sm: int = 132, target_dtype: torch.dtype = torch.int64) -> dict:
    """The launch path of one call as a dict.

    kernel   "sigmoid" (n scores), "softmax" (n rows of c), "fused" (K11: n rows of c, `target_dtype` labels)
    binding  "ctypes" (`_native`: scratch entries), "torch" (the registered operator: scratch-less entries) or "abi" (a
             scratch entry called directly with `scratch` = "owned" | "short" (softmax: fewer than 8 + n bytes) |
             "misaligned" (not 4-byte aligned))
    offset   the input's element offset from a 16-byte boundary (a sliced view)

    sigmoid: small (one CTA), flag (range_flag_kernel + sigmoid_if_kernel: grid, the aligned body's vectors, the scalar head
    and tail) or spec (sigmoid_spec_kernel + fix-up: tiles, the tail-only extra tile, grid, tiles per CTA, scalar tail).
    softmax: spec (softmax_spec_kernel + fix-up: kIter, grid, rows per warp) or flag (range_flag_kernel + softmax_if_kernel).
    fused: stats_softmax_kernel (kIter, the target load, grid, rows per warp) + restore_if_not_logits_kernel."""
    esize = torch.empty(0, dtype=dtype).element_size()
    f64 = dtype == torch.float64
    if kernel == "sigmoid":
        if n <= (SMALL_N_F64 if f64 else SMALL_N):
            return dict(kernel="small", grid=1)
        grid = min(_cdiv(n, 2048), sm * 8)
        spec = (binding != "torch" and not f64 and (offset * esize) % 16 == 0 and scratch == "owned")
        if not spec:
            if f64:
                return dict(kernel="flag", grid=grid, head=0, vectors=0, tail=n)
            kvec = 16 // esize
            head = min((kvec - offset % kvec) % kvec, n)
            nvec = (n - head) // kvec
            return dict(kernel="flag", grid=grid, head=head, vectors=nvec, tail=n - head - nvec * kvec)
        kvec = 16 // esize
        nvec = n // kvec
        extra = nvec % TILE_VECS == 0 and n % kvec != 0
        tiles = _cdiv(nvec, TILE_VECS) + int(extra)
        grid = min(tiles, sm * 8)
        return dict(kernel="spec", tiles=tiles, extra_tile=extra, grid=grid, tiles_per_cta=_cdiv(tiles, grid), tail=n % kvec)
    kiter = 1 << max(0, math.ceil(math.log2(_cdiv(min(c, 1024), 32))))
    if kernel == "fused":
        grid = max(1, min(_cdiv(n, 8), sm * 3))
        return dict(kernel="fused", kiter=kiter, load="kI64" if target_dtype == torch.int64 else "load_label", grid=grid,
                    rows_per_warp=_cdiv(n, grid * 8))
    spec = binding != "torch" and not f64 and c <= 1024 and scratch == "owned"
    if spec:
        grid = min(_cdiv(n, 8), sm * 3)
        return dict(kernel="spec", kiter=kiter, grid=grid, rows_per_warp=_cdiv(n, grid * 8))
    grid = min(_cdiv(n, 8), sm * 8)
    return dict(kernel="flag", grid=grid, rows_per_warp=_cdiv(n, grid * 8))
