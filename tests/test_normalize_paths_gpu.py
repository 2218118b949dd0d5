"""GPU: logit normalisation (K6: `normalize_logits_if_needed`, csrc/curve.cu) and the softmax of the fused stats update
(K11, csrc/fused.cu) against the reference's chain restated in torch (oracle/normalize.py `chain`) on the same GPU, and
against an exact evaluation (`exact`, numpy, float64 or wider) within a derived forward-error bound (`bound`), on every
launch path and binding:
  paths     sigmoid: the one-CTA kernel (n <= 32768, float64 n <= 12288); the vote + apply pair (range_flag_kernel,
            sigmoid_if_kernel: float64, views misaligned by every element offset, the scratch-less entry of the torch
            binding, an unaligned caller scratch); the speculative single pass with its fix-up launch.  softmax: the
            speculative row kernel at every kIter bucket edge; the vote + three-pass row kernel (C > 1024, float64, the torch
            binding, a caller scratch shorter than 8 + n).  K11: every kIter edge, int64 targets and the four narrower integer
            dtypes, micro and macro; float64 is rejected
  geometry  n = 32768 / 32769, tile multiples and +-1, a whole number of tiles plus a scalar tail (the extra tile), more
            tiles than the sigmoid grid (1056 CTAs) and more rows than the softmax / K11 grid has warps (3168); one float16
            sigmoid and one float16 softmax of more than 2^31 elements
  votes     logits, probabilities, and one out-of-range score at the first / last element, the first / last element of a
            tile, only in the scalar tail, only in the misaligned head, in a row of a warp that already voted
  values    every float16 / bfloat16 bit pattern on each sigmoid path; float32 ulp windows at 0 and the subnormals, at
            +-88.72 (expf overflows), near +-103.97 (subnormal sigmoids), where the sigmoid rounds to 1, at +-inf; float64
            windows at +-709.78 and +-745.13; softmax rows with ties, +inf, all -inf, NaN in the first / last column, +-0, a
            +-1e30 spread; probability batches holding -0.0, subnormals and NaN
Every case first asserts its path with `path_of`.  The bars: bit equality with `chain` for every sigmoid, for the softmax in
float32 / float16 / bfloat16 with C <= 1024 and in float64 with C <= 512 (ATen's warp-softmax range), and for K11's
probabilities, which also equal K6's; NaN only needs to be NaN where arithmetic made it, and a batch that is passed through
keeps its bits, NaN payloads included, except on the speculative softmax's write-through (T -> float -> T), which keeps
NaN-ness only.  Every output lies within `bound` of `exact` (all of C > 1024, float64 C > 512 and N-d inputs included).
K11's tp / fp / tn / fn equal oracle/multiclass_counts.py's chain over the admitted rows after each of two updates, its
workspace is zero after each, and an out-of-range target raises MB200_FLAG_TARGET_RANGE without being counted.
Outputs written through the C-ABI start out as a NaN sentinel and the caller scratch as stale bytes.
"""
import contextlib
import math

import pytest
import torch

from metrics_b200 import _native
from oracle import multiclass_counts as om
from oracle import normalize as on

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F16, BF16, F32, F64 = torch.float16, torch.bfloat16, torch.float32, torch.float64
NAN, INF = float("nan"), float("inf")
INT_VIEW = {8: torch.int64, 4: torch.int32, 2: torch.int16}
SENTINEL = {F32: 0x7FC05A5A, F16: 0x7E5A, BF16: 0x7FDA, F64: 0x7FF8000000005A5A}
TILE = {F32: 4096, F16: 8192, BF16: 8192}  # elements of one speculative sigmoid tile (16 KB)
KVEC = {F32: 4, F16: 8, BF16: 8, F64: 2}
SOFTMAX_C = [1, 2, 31, 32, 33, 64, 65, 128, 129, 256, 257, 512, 513, 1023, 1024]
WIDE_C = [1025, 2048, 4096]


def sm():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def rows_per_wave():
    """Warps of the speculative softmax / K11 grid (3 CTAs of 8 warps per SM): 3168 on an H100 SXM."""
    return sm() * 3 * 8


def path(kernel, x, c=1, **kw):
    n = x.numel() // c
    offset = (x.data_ptr() % 16) // x.element_size()
    return on.path_of(kernel, x.dtype, n, c, offset=offset, sm=sm(), **kw)


def expect(p, want):
    for k, v in want.items():
        assert (v(p[k]) if callable(v) else p[k] == v), (k, p[k], v, p)


def bits(t):
    return t.view(INT_VIEW[t.element_size()])


def sentinel_like(x):
    out = torch.empty_like(x, memory_format=torch.contiguous_format)
    bits(out).fill_(SENTINEL[x.dtype])
    return out


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def logits(n, dtype, seed, scale=5.0):
    return (torch.randn(n, generator=gen(seed), device=DEV, dtype=F32) * scale).to(dtype)


def probs(n, dtype, seed):
    return torch.rand(n, generator=gen(seed), device=DEV, dtype=F32).to(dtype)


@contextlib.contextmanager
def binding(name):
    old = _native._TORCH_BINDING
    _native._TORCH_BINDING = name == "torch"
    try:
        yield
    finally:
        _native._TORCH_BINDING = old


def abi_sigmoid(x, scratch="owned"):
    """`mb200_curve_sigmoid_if_logits_scratch` on a sentinel output and a scratch of stale bytes (`misaligned`: 1 byte off)."""
    out = sentinel_like(x)
    n = x.numel()
    nb = int(_native.lib().mb200_curve_normalize_scratch_bytes(n))
    buf = torch.full((nb + 8,), 0xAB, dtype=torch.uint8, device=DEV)
    sp = buf.data_ptr() + (1 if scratch == "misaligned" else 0)
    _native.check(_native.lib().mb200_curve_sigmoid_if_logits_scratch(x.data_ptr(), _native.tag(x), n, out.data_ptr(), sp, nb,
                                                                       _native.stream_handle(x.device)), "sigmoid_if_logits_scratch")
    return out


def abi_softmax(x, scratch="owned"):
    """`mb200_curve_softmax_if_logits_scratch` on `[n, c]` with a sentinel output; `short`: one byte less than 8 + n."""
    out = sentinel_like(x)
    n, c = x.shape
    nb = 8 + n - (1 if scratch == "short" else 0)
    buf = torch.full((nb + 8,), 0xAB, dtype=torch.uint8, device=DEV)
    sp = buf.data_ptr() + (1 if scratch == "misaligned" else 0)
    _native.check(_native.lib().mb200_curve_softmax_if_logits_scratch(x.data_ptr(), _native.tag(x), n, c, out.data_ptr(), sp, nb,
                                                                       _native.stream_handle(x.device)), "softmax_if_logits_scratch")
    return out


def run(norm, x, via):
    if via in ("ctypes", "torch"):
        with binding(via):
            return _native.sigmoid_if_logits(x) if norm == "sigmoid" else _native.softmax_if_logits(x)
    scratch = via.split("_", 1)[1] if "_" in via else "owned"
    return abi_sigmoid(x, scratch) if norm == "sigmoid" else abi_softmax(x, scratch)


def assert_same(got, want, case, strict_nan):
    """Bit equality; where `want` is NaN, NaN-ness only unless `strict_nan` (a pass-through keeps payloads)."""
    assert got.dtype == want.dtype and got.shape == want.shape, case
    nan_w = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan_w), (case, "NaN positions differ")
    same = bits(got) == bits(want)
    if not strict_nan:
        same |= nan_w
    if not bool(same.all()):
        i = int((~same).flatten().nonzero()[0])
        raise AssertionError((case, int((~same).sum()), "first at", i, float(got.flatten()[i]), float(want.flatten()[i])))


def assert_bound(got, x, norm, case):
    nbad, worst = on.violations(got, x, norm)
    assert nbad == 0, (case, worst)


def verify(norm, x, vias, case, bitwise=True, exact=True):
    """Run `x` through each binding / entry of `vias` ({via: expected path fields}); compare with `chain` and `exact`."""
    c = x.shape[1] if norm == "softmax" else 1
    want = on.chain(x, norm) if bitwise else None
    is_logits = on.is_logits(x)
    for via, fields in vias.items():
        kw = dict(binding="torch" if via == "torch" else ("ctypes" if via == "ctypes" else "abi"),
                  scratch=via.split("_", 1)[1] if "_" in via else "owned")
        rows = x if x.ndim <= 2 else x.movedim(1, -1).reshape(-1, c)
        p = path(norm, rows, c, **kw)
        expect(p, fields)
        got = run(norm, x, via)
        assert got.shape == x.shape and got.dtype == x.dtype and got.is_contiguous(), (case, via)
        if bitwise:
            strict = not is_logits and not (norm == "softmax" and p["kernel"] == "spec")
            assert_same(got, want, (case, via, p), strict)
        elif not is_logits:  # N-d pass-through: the input's bits
            assert_same(got, x.contiguous(), (case, via, p), p["kernel"] != "spec")
        if exact:
            assert_bound(got, x, norm, (case, via, p))


def votes(n, tile, kvec, offset=0):
    """Index of the single out-of-range score for each placement that exists at this n."""
    v = {"first": 0, "last": n - 1}
    if n > tile:
        v["tile_first"], v["tile_last"] = tile, tile - 1
    head = (kvec - offset % kvec) % kvec
    if offset and head:
        v["head_only"] = head - 1
    tail = (n - head) % kvec
    if tail:
        v["tail_only"] = n - tail
    return v


def with_vote(x, i, value=-0.25):
    y = x.clone()
    y.view(-1)[i] = value
    return y


# ------------------------------------------------------------------------------------------------------------------
# sigmoid
# ------------------------------------------------------------------------------------------------------------------
SIG_GEOMETRY = [(F32, 32768), (F32, 32769), (F32, 4096 * 9), (F32, 4096 * 9 - 1), (F32, 4096 * 9 + 1), (F32, 4096 * 12 + 3),
                (F16, 32769), (F16, 8192 * 5), (F16, 8192 * 5 - 1), (F16, 8192 * 5 + 1), (F16, 8192 * 6 + 7),
                (BF16, 32768), (BF16, 8192 * 5 + 1), (BF16, 8192 * 6 + 5), (F32, (1 << 23) + 3),
                (F64, 12288), (F64, 12289), (F64, 100003)]


def sigmoid_vias(dtype, n):
    small = n <= (on.SMALL_N_F64 if dtype == F64 else on.SMALL_N)
    if small:
        return {v: {"kernel": "small"} for v in ("ctypes", "torch", "abi")}
    big = {"kernel": "spec" if dtype != F64 else "flag"}
    return {"ctypes": big, "abi": big, "torch": {"kernel": "flag"}, "abi_misaligned": {"kernel": "flag"}}


@pytest.mark.parametrize("dtype,n", SIG_GEOMETRY, ids=lambda v: str(v))
def test_sigmoid_geometry_and_votes(dtype, n):
    vias = sigmoid_vias(dtype, n)
    spec = vias["ctypes"]["kernel"] == "spec"
    if spec:
        p = path("sigmoid", torch.empty(n, dtype=dtype, device=DEV))
        assert p["extra_tile"] == (n // KVEC[dtype] % 1024 == 0 and n % KVEC[dtype] != 0)
        if n > (1 << 23):
            assert p["tiles"] > sm() * 8 and p["tiles_per_cta"] >= 2
    seed = n % 1000
    verify("sigmoid", logits(n, dtype, seed), vias, (dtype, n, "logits"))
    base = probs(n, dtype, seed + 1)
    verify("sigmoid", base, vias, (dtype, n, "probs"))
    for name, i in votes(n, TILE.get(dtype, 1 << 30), KVEC[dtype]).items():
        for value in ((-0.25, 1.5) if n < (1 << 20) else (-0.25,)):
            verify("sigmoid", with_vote(base, i, value), vias, (dtype, n, name, value))


@pytest.mark.parametrize("dtype", [F32, F16, BF16])
def test_sigmoid_misaligned_views(dtype):
    """`preds[k:]` of an aligned buffer keeps its offset through `.contiguous()`: every offset 1..kVec-1 takes the vote +
    apply pair; a single logit in the misaligned head alone, or in the scalar tail alone, decides the batch."""
    n = 70001
    for k in range(1, KVEC[dtype]):
        buf = probs(n + k, dtype, k)
        x = buf[k:]
        assert (x.data_ptr() % 16) // x.element_size() == k
        p = path("sigmoid", x)
        expect(p, {"kernel": "flag", "head": KVEC[dtype] - k})
        vias = {"ctypes": {"kernel": "flag"}, "torch": {"kernel": "flag"}, "abi": {"kernel": "flag"}}
        verify("sigmoid", x, vias, (dtype, k, "probs"))
        for name, i in votes(n, TILE[dtype], KVEC[dtype], offset=k).items():
            y = buf.clone()
            y[k + i] = 1.75
            verify("sigmoid", y[k:], vias, (dtype, k, name))
        assert "head_only" in votes(n, TILE[dtype], KVEC[dtype], offset=k)


@pytest.mark.parametrize("dtype", [F16, BF16])
@pytest.mark.parametrize("kernel", ["small", "flag", "spec"])
def test_sigmoid_every_bit_pattern(dtype, kernel):
    every = torch.arange(-32768, 32768, dtype=torch.int32, device=DEV).to(torch.int16).view(dtype)
    if kernel == "small":
        for half in every.chunk(2):
            verify("sigmoid", half, {"ctypes": {"kernel": "small"}, "torch": {"kernel": "small"}}, (dtype, kernel))
        return
    if kernel == "flag":
        buf = torch.zeros(every.numel() + 3, dtype=dtype, device=DEV)
        buf[3:] = every
        x = buf[3:]
        verify("sigmoid", x, {"ctypes": {"kernel": "flag"}, "torch": {"kernel": "flag"}, "abi_misaligned": {"kernel": "flag"}},
               (dtype, kernel))
        return
    verify("sigmoid", every, {"ctypes": {"kernel": "spec", "tiles": 8}, "abi": {"kernel": "spec"}}, (dtype, kernel))


def ulp_window(center, k, dtype):
    """`center` rounded to dtype (float32 / float64) and its k neighbours on each side, walking through zero and the
    subnormals to the other sign; NaN patterns beyond +-inf are left out."""
    nbits = 64 if dtype == F64 else 32
    sign = 1 << (nbits - 1)
    b = bits(torch.tensor(center, dtype=dtype)).item()
    o = b if b >= 0 else -(b & (sign - 1))  # position on the number line, in ulps (-0.0 and +0.0 share 0)
    pats = [(j if j >= 0 else (-j) | sign) for j in range(o - k, o + k + 1)]
    w = torch.tensor([u - (1 << nbits) if u >= sign else u for u in pats], dtype=INT_VIEW[nbits // 8]).view(dtype)
    return w[~torch.isnan(w)]


@pytest.mark.parametrize("dtype", [F32, F64])
def test_sigmoid_ulp_windows(dtype):
    if dtype == F32:
        centers = [0.0, -0.0, 1e-40, -1e-40, 88.72, -88.72, 103.97, -103.97, 16.635532, 17.0, -16.635532, 3.4028235e38, -3.4028235e38]
        k = 1000
    else:
        centers = [709.78, -709.78, 745.13, -745.13, 36.7368, -36.7368]
        k = 900
    w = torch.cat([ulp_window(c, k, dtype) for c in centers] + [torch.tensor([INF, -INF, 0.5], dtype=dtype)]).to(DEV)
    assert w.numel() <= (on.SMALL_N_F64 if dtype == F64 else on.SMALL_N)
    verify("sigmoid", w, {"ctypes": {"kernel": "small"}, "torch": {"kernel": "small"}}, (dtype, "small"))
    pad = torch.cat([w, w, w]) if dtype == F64 else torch.cat([w, probs(40000 - w.numel(), dtype, 3)])
    verify("sigmoid", pad, sigmoid_vias(dtype, pad.numel()), (dtype, "large"))


def test_sigmoid_f16_beyond_2_31_elements():
    """2^31 + 5 float16 probabilities with one logit in the scalar tail: every one of the 262145 tiles is pending and the
    fix-up launch revisits them all.  Compared in chunks; the buffers are freed at the end."""
    n = (1 << 31) + 5
    expect(on.path_of("sigmoid", F16, n, sm=sm()), {"kernel": "spec", "tiles": 262145, "extra_tile": True, "tail": 5})
    x = torch.empty(n, dtype=F16, device=DEV)
    x.uniform_(0, 1, generator=gen(31))
    x[n - 2] = -3.0  # in the scalar tail
    try:
        got = _native.sigmoid_if_logits(x)
        step = 1 << 27
        for s in range(0, n, step):
            assert torch.equal(bits(got[s:s + step]), bits(torch.sigmoid(x[s:s + step]))), s
        idx = torch.randint(0, n, (1 << 20,), generator=gen(32), device=DEV)
        idx[:3] = torch.tensor([0, n - 2, n - 1], device=DEV)
        assert_bound(got[idx], x[idx], "sigmoid", "f16 > 2^31 sample")
        del got
    finally:
        del x
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# softmax
# ------------------------------------------------------------------------------------------------------------------
def softmax_probs(n, c, dtype, seed):
    return torch.softmax(torch.randn(n, c, generator=gen(seed), device=DEV), 1).to(dtype)


def softmax_vias(dtype, c):
    spec = dtype != F64 and c <= 1024
    return {"ctypes": {"kernel": "spec" if spec else "flag"}, "torch": {"kernel": "flag"},
            "abi_short": {"kernel": "flag"}, "abi_misaligned": {"kernel": "flag"}}


@pytest.mark.parametrize("dtype", [F32, F16, BF16, F64])
@pytest.mark.parametrize("c", SOFTMAX_C + WIDE_C)
def test_softmax_kiter_edges_and_votes(dtype, c):
    rows = rows_per_wave()
    n = rows + 37 if c <= 256 else 300
    vias = softmax_vias(dtype, c)
    if vias["ctypes"]["kernel"] == "spec":
        expect(on.path_of("softmax", dtype, n, c, sm=sm()),
               {"kiter": 1 << max(0, math.ceil(math.log2(-(-c // 32)))), "rows_per_warp": 2 if n > rows else 1})
    bitwise = (dtype != F64 and c <= 1024) or (dtype == F64 and c <= 512)
    x = (torch.randn(n, c, generator=gen(c), device=DEV) * 3).to(dtype)
    verify("softmax", x, vias, (dtype, c, "logits"), bitwise=bitwise)
    base = softmax_probs(n, c, dtype, c + 1)
    verify("softmax", base, vias, (dtype, c, "probs"), bitwise=True)
    places = {"first": (0, 0), "last": (n - 1, c - 1), "second_row_of_warp_0": (min(rows, n - 1), c // 2)}
    if n > rows:
        places["first_row_of_a_warp_with_a_second"] = (5, 0)
    for name, (r, col) in places.items():
        y = base.clone()
        y[r, col] = -2.0
        verify("softmax", y, vias, (dtype, c, name), bitwise=bitwise)


@pytest.mark.parametrize("dtype", [F32, F16, BF16, F64])
@pytest.mark.parametrize("c", [37, 1500])
def test_softmax_special_rows(dtype, c):
    """Ties, one +inf (the row is NaN, as in ATen), all -inf (NaN), NaN in the first / last column (NaN), +-0, a +-1e30
    spread (+-inf in float16: NaN rows); then probability batches holding -0.0, subnormals and NaN, passed through."""
    n = 64
    x = (torch.randn(n, c, generator=gen(c + 7), device=DEV) * 2).to(dtype)
    x[0] = 2.0
    x[1, : c // 2] = 1.5
    x[2, 3] = INF
    x[3] = -INF
    x[4, 0] = NAN
    x[5, c - 1] = NAN
    x[6] = 0.0
    x[6, 1::2] = -0.0
    x[7, 0], x[7, 1] = -1e30, 1e30
    x[8, :] = -1e30
    x[8, c - 1] = 1e30
    bitwise = c <= (512 if dtype == F64 else 1024)
    verify("softmax", x, softmax_vias(dtype, c), (dtype, c, "special"), bitwise=bitwise)
    p = softmax_probs(n, c, dtype, c + 8)
    p[0, 0] = -0.0
    p[1, 1] = torch.finfo(dtype).tiny / 4 if dtype != F16 else 2.0 ** -24
    p[2, 2] = NAN
    p[3, c - 1] = NAN
    bits(p)[4, 3] = {F32: 0x7FC01234, F16: 0x7E12, BF16: 0x7FD2, F64: 0x7FF8000000001234}[dtype]  # a NaN payload
    verify("softmax", p, softmax_vias(dtype, c), (dtype, c, "special probs"), bitwise=True)


@pytest.mark.parametrize("dtype", [F32, F16, BF16, F64])
@pytest.mark.parametrize("shape", [(6, 11, 7), (4, 40, 3, 5), (2, 1100, 3), (3, 1, 4)])
def test_softmax_nd(dtype, shape):
    """An `[N, C, d...]` input is normalised over dim 1 on both bindings, every element written, the vote taken over every
    element (a single logit in the last element, beyond the first N * C, decides); held to the exact bound."""
    c = shape[1]
    vias = {"ctypes": softmax_vias(dtype, c)["ctypes"], "torch": {"kernel": "flag"}}
    x = (torch.randn(*shape, generator=gen(sum(shape)), device=DEV) * 3).to(dtype)
    verify("softmax", x, vias, (dtype, shape, "logits"), bitwise=False)
    got = _native.softmax_if_logits(x)
    want = torch.softmax(x.double(), 1)
    assert float((got.double() - want).abs().max()) < (1e-2 if dtype in (F16, BF16) else 1e-5)
    p = torch.softmax(torch.randn(*shape, generator=gen(3), device=DEV), 1).to(dtype)
    verify("softmax", p, vias, (dtype, shape, "probs"), bitwise=False)
    q = p.clone()
    q.view(-1)[-1] = 1.25
    verify("softmax", q, vias, (dtype, shape, "last element"), bitwise=False)


def test_softmax_f16_beyond_2_31_elements():
    """2^21 + 1 rows of 1024 float16 logits (2^31 + 1024 scores) on the speculative kernel, compared in row chunks."""
    n, c = (1 << 21) + 1, 1024
    expect(on.path_of("softmax", F16, n, c, sm=sm()), {"kernel": "spec", "kiter": 32})
    x = torch.empty(n, c, dtype=F16, device=DEV)
    x.normal_(0, 3, generator=gen(41))
    try:
        got = _native.softmax_if_logits(x)
        step = 1 << 17
        for s in range(0, n, step):
            assert torch.equal(bits(got[s:s + step]), bits(torch.softmax(x[s:s + step], 1))), s
        rows = torch.tensor([0, 1, n // 2, n - 2, n - 1], device=DEV)
        assert_bound(got[rows], x[rows], "softmax", "f16 > 2^31 sample rows")
        del got
    finally:
        del x
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# K11: fused stat scores + softmax
# ------------------------------------------------------------------------------------------------------------------
TARGETS = [torch.int64, torch.int32, torch.int16, torch.int8, torch.uint8]


def fused_case(n, c, dtype, tdtype, seed, kind="logits"):
    g = gen(seed)
    if kind == "logits":
        x = (torch.randn(n, c, generator=g, device=DEV) * 3).to(dtype)
    else:
        x = softmax_probs(n, c, dtype, seed)
    hi = min(c, torch.iinfo(tdtype).max + 1)
    t = torch.randint(0, hi, (n,), generator=g, device=DEV).to(tdtype)
    return x, t


def bad_label(tdtype, c):
    return -1 if tdtype != torch.uint8 else (c if c <= 255 else None)


FUSED_CASES = ([("ctypes", c, torch.int64) for c in SOFTMAX_C]
               + [("ctypes", c, td) for td in TARGETS[1:] for c in (1, 33, 129, 513, 1024)]
               + [("torch", c, torch.int64) for c in (1, 33, 129, 513, 1024)] + [("torch", 65, torch.int32)])


@pytest.mark.parametrize("via,c,tdtype", FUSED_CASES, ids=lambda v: str(v))
@pytest.mark.parametrize("dtype", [F32, F16, BF16])
@pytest.mark.parametrize("micro", [False, True])
def test_fused_stats_softmax(micro, dtype, via, c, tdtype):
    """Every kIter edge with int64 targets, the narrower target dtypes at one C per bucket, the torch binding."""
    rows = rows_per_wave()
    n = rows + 41 if c <= 129 else 257
    p = on.path_of("fused", dtype, n, c, sm=sm(), target_dtype=tdtype)
    expect(p, {"load": "kI64" if tdtype == torch.int64 else "load_label"})
    if n > rows:
        assert p["rows_per_warp"] == 2
    for kind in ("logits", "probs", "mixed"):
        x, t = fused_case(n, c, dtype, tdtype, c * 3 + len(kind), "logits" if kind == "logits" else "probs")
        if kind == "mixed":
            x[rows % n, c // 2] = 1.5  # one logit row in a warp's second round: every row written so far must be redone
        bad = bad_label(tdtype, c)
        if bad is not None:
            t[3] = bad
            t[n - 1] = bad
        valid = (t.long() >= 0) & (t.long() < c)
        want = om.stat_scores(x[valid], t[valid].long(), c, 1, "micro" if micro else "none", "global", None).reshape(4, -1)
        states = [torch.zeros(1 if micro else c, dtype=torch.int64, device=DEV) for _ in range(4)]
        ws = torch.zeros(3 * c + 2, dtype=torch.int64, device=DEV)
        flag = torch.zeros(1, dtype=torch.int32, device=DEV)
        chain = on.chain(x, "softmax")
        k6 = _native.softmax_if_logits(x)
        for rep in (1, 2):
            with binding(via):
                probs = _native.multiclass_stats_softmax_update_(*states, ws, x, t, c, micro, flag)
            assert int(flag.item()) == (_native.FLAG_TARGET_RANGE if bad is not None else 0), (kind, rep)
            assert not bool(ws.any()), (kind, rep, "workspace left dirty")
            got = torch.stack(states)
            assert torch.equal(got, rep * want), (via, dtype, c, tdtype, micro, kind, rep, (got - rep * want).abs().sum(-1).tolist())
            assert_same(probs, chain, (via, dtype, c, kind, "chain"), strict_nan=not on.is_logits(x))
            assert_same(probs, k6, (via, dtype, c, kind, "K6"), strict_nan=False)
            assert_bound(probs, x, "softmax", (via, dtype, c, kind))


def test_fused_restore_keeps_every_bit():
    """A probability batch holding -0.0, a subnormal and NaN payloads is stored as it is (the restore kernel copies bits)."""
    n, c = rows_per_wave() + 9, 65
    x, t = fused_case(n, c, F32, torch.int64, 77, "probs")
    x[0, 0] = -0.0
    x[1, 1] = 1e-40
    bits(x)[2, 2] = 0x7FC01234
    bits(x)[n - 9, 3] = 0x7FA00001  # a signalling NaN pattern
    states = [torch.zeros(c, dtype=torch.int64, device=DEV) for _ in range(4)]
    ws = torch.zeros(3 * c + 2, dtype=torch.int64, device=DEV)
    probs = _native.multiclass_stats_softmax_update_(*states, ws, x, t, c, False)
    assert torch.equal(bits(probs), bits(x))


def test_fused_rejects_float64():
    x = torch.rand(10, 4, dtype=F64, device=DEV)
    t = torch.zeros(10, dtype=torch.int64, device=DEV)
    states = [torch.zeros(4, dtype=torch.int64, device=DEV) for _ in range(4)]
    ws = torch.zeros(3 * 4 + 2, dtype=torch.int64, device=DEV)
    out = torch.empty_like(x)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    rc = _native.lib().mb200_multiclass_stats_softmax_update(
        x.data_ptr(), _native.tag(x), t.data_ptr(), _native.tag(t), 10, 4, 0, *(s.data_ptr() for s in states), ws.data_ptr(),
        out.data_ptr(), flag.data_ptr(), None, _native.stream_handle(x.device))
    assert rc == -1 and "f32/f16/bf16" in _native.lib().mb200_last_error().decode()
    with pytest.raises(ValueError, match="f32/f16/bf16"):
        _native.multiclass_stats_softmax_update_(*states, ws, x, t, 4, False)
