"""GPU: kernels K1 / K1b (`mb200_multiclass_confmat_update`, `mb200_multiclass_stat_scores_update`, `..._topk_update`,
`..._samplewise`, `mb200_argmax_rows`; csrc/confmat.cu) against the reference's own chain of torch ops
(oracle/multiclass_counts.py) run on the same GPU, bit for bit, on every launch path and sink of `confmat.cu`:

  kernels  vec (warp per row, 16-byte loads, programmatic dependent launch for the confusion-matrix and deferred sinks),
           scalar (float64, odd row bytes, misaligned base), strided (C < 32, `[N, C, d...]`), labels (integer
           predictions), top-k
  sinks    confusion matrix in shared memory / global; stat scores in shared memory / global / deferred fold, micro and
           macro; samplewise; argmax

Every case first asserts its path with `path_of`, which restates the dispatch, so a change to the dispatch fails here
instead of leaving a path untested.  Every accumulating case runs two updates into the same state and expects twice the
chain, checks that the stat-score workspace is zero after each call, and that the error word is set exactly when a target
outside `[0, C)` is not ignored (the kernel then skips that row; the chain is run on the other rows).

The rows hold what argmax kernels get wrong: the maximum at column 0, at C - 1, inside the last vector and on both sides of
each 2 KiB chunk edge (512 float32 / 1024 half-precision columns); duplicate maxima later in the vector, in another lane and
in a later chunk; NaN alone, beside a larger value, in two chunks and with a negative-sign payload; all -inf, -0 before +0,
a subnormal maximum among zeros and all-equal rows; and every float16 / bfloat16 bit pattern as some row's maximum.

`ignore_index` is compared as the reference compares it: ATen casts the Python int to the target's dtype, so with uint8
targets 257 drops class 1 and -1 drops 255.
"""
import pytest
import torch

from metrics_b200 import _native
from oracle import multiclass_counts as om

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FLOATS = [torch.float32, torch.float16, torch.bfloat16]
# (520 and 1032: one vector past a chunk edge with 16-byte rows in every dtype; 511 / 513 / 1023 ... take the scalar path)
SIZES = [1, 2, 31, 32, 33, 63, 64, 65, 255, 256, 257, 511, 512, 513, 520, 1000, 1023, 1024, 1025, 1032, 2047, 2048, 2049,
         4100]
LABEL_DTYPES = [torch.int8, torch.uint8, torch.int16, torch.int32, torch.int64]


# ------------------------------------------------------------------------------------------------------------------
# the dispatch of confmat.cu, restated
# ------------------------------------------------------------------------------------------------------------------
def geometry(preds, target):
    if preds.ndim == target.ndim + 1:
        inner = 1
        for s in preds.shape[2:]:
            inner *= s
        return True, preds.shape[0], inner
    return False, preds.numel(), 1


def path_of(entry, preds, target, num_classes, micro=False):
    """(kernel, sink) that `entry` launches: kernel in vec (programmatic launch) / vec_plain / scalar / strided / labels /
    topk."""
    C = num_classes
    class_dim, n_outer, inner = geometry(preds, target)
    total = n_outer * inner
    if entry == "confmat":
        sink = "confmat_smem" if C * C <= 4096 and total >= 4096 else "confmat_global"
    elif entry == "stats":
        if not micro and C <= 256 and total >= 4096 and total >= 16 * C:
            sink = "stats_smem"
        elif class_dim and inner == 1 and n_outer * C >= 1 << 24:
            sink = "stats_deferred"
        else:
            sink = "stats_global"
    elif entry == "topk":
        return "topk", "stats_global"
    else:
        sink = entry  # samplewise, argmax
    if not class_dim:
        return "labels", sink
    if inner != 1 or C < 32:
        return "strided", sink
    item = preds.element_size()
    if not (item <= 4 and (C * item) % 16 == 0 and preds.data_ptr() % 16 == 0):
        return "scalar", sink
    if sink in ("confmat_smem", "confmat_global", "stats_deferred"):
        return "vec", sink
    return "vec_plain", sink


# ------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------
NEG_NAN_BITS = {torch.float32: (torch.int32, -4194303), torch.float16: (torch.int16, -511),
                torch.bfloat16: (torch.int16, -63), torch.float64: (torch.int64, -2251799813685247)}
SUBNORMAL = {torch.float32: 2.0**-149, torch.float16: 2.0**-24, torch.bfloat16: 2.0**-133, torch.float64: 5e-324}
N_KINDS = 14


def chunk_cols(dtype) -> int:
    return 2048 // torch.tensor([], dtype=dtype).element_size()


def rows(n: int, C: int, dtype, seed: int = 0) -> torch.Tensor:
    """`[n, C]` scores on the device; row r is of kind r % 14 (see the module docstring), at random columns."""
    g = torch.Generator().manual_seed(seed * 7919 + C)
    x = torch.randn(n, C, generator=g, dtype=torch.float64)
    epv, E = 16 // torch.tensor([], dtype=dtype).element_size(), chunk_cols(dtype)
    r = torch.arange(n)
    kind, lap = r % N_KINDS, r // N_KINDS  # lap alternates the variants of one kind
    j = torch.randint(0, C, (n,), generator=g)
    top = float(x.abs().max()) + 2

    def put(k, cols, val):
        m = kind == k
        x[r[m], cols[m].clamp(0, C - 1)] = val

    zero = torch.zeros(n, dtype=torch.long)
    put(1, zero, top)
    put(2, zero + C - 1, top)
    put(3, C - 1 - j % epv, top)  # inside the last (clamp-duplicated) vector
    edge = E * (1 + j % max(1, (C - 1) // E))
    put(4, edge - 1 + lap % 2, top)  # either side of a chunk edge
    j0 = j % max(1, C // 2)
    put(5, j0 + torch.tensor([1, epv, E])[lap % 3], top)  # a duplicate later in the vector / in another lane / chunk
    put(5, j0, top)
    put(6, j, float("nan"))
    put(7, j + 1 - 2 * (lap % 2), top + 1)  # a larger finite value beside the NaN
    put(7, j, float("nan"))
    put(8, j % E, float("nan"))
    put(8, j % E + E, float("nan"))
    put(9, j, float("nan"))  # its bits become a negative-sign payload below
    x[kind == 10] = float("-inf")
    m11 = kind == 11
    x[m11] = -1.0
    put(11, j + 1 + lap % 5, 0.0)
    put(11, j, -0.0)  # -0 first: it must win the tie with the later +0
    m12 = kind == 12
    x[m12] = torch.where(lap[m12, None] % 2 == 0, 0.0, -0.0).double()
    put(12, j, SUBNORMAL[dtype])
    x[kind == 13] = x[kind == 13][:, :1]
    y = x.to(dtype)
    itype, bits = NEG_NAN_BITS[dtype]
    m9 = kind == 9
    y.view(itype)[r[m9], j[m9]] = bits
    return y.to(DEV)


def stored(value: int, dtype) -> int:
    """What `value` becomes in a tensor of `dtype` (two's complement wrap, as ATen casts a Python int)."""
    return int(torch.tensor([value], dtype=torch.int64).to(dtype).item())


def targets(n, C, dtype=torch.int64, ignore_index=None, seed=1, bad=()):
    """`[n]` labels in [0, C); an eighth hold `ignore_index` (as the dtype stores it); rows in `bad` hold a label outside
    [0, C) that is not ignored."""
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, C, (n,), generator=g)
    if ignore_index is not None:
        t[torch.rand(n, generator=g) < 0.125] = stored(ignore_index, dtype)
    for r in bad:
        t[r] = next(v for v in (C, C + 1, -2, -3) if stored(v, dtype) == v
                    and (ignore_index is None or v != stored(ignore_index, dtype)))
    return t.to(dtype).to(DEV)


def misaligned(x: torch.Tensor) -> torch.Tensor:
    """A contiguous copy of x whose base is one element past a 16-byte boundary."""
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device=x.device)
    v = buf[1:].view(x.shape)
    v.copy_(x)
    assert v.data_ptr() % 16 != 0 and v.is_contiguous()
    return v


# ------------------------------------------------------------------------------------------------------------------
# kernel vs chain
# ------------------------------------------------------------------------------------------------------------------
def admitted(preds, target, C, ignore_index):
    """(preds, target, any bad): the rows the kernel counts.  A target outside [0, C) that is not ignored (compared in the
    target's dtype) is flagged and skipped; the chain cannot take it, so it gets the other rows, flattened to `[M, C]`."""
    ign = torch.zeros_like(target, dtype=torch.bool) if ignore_index is None else target == ignore_index
    tl = target.long()
    bad = ~ign & ((tl < 0) | (tl >= C))
    if not bool(bad.any()):
        return preds, target, False
    keep = ~bad.flatten()
    if preds.ndim == target.ndim + 1:
        p = preds.movedim(1, -1).reshape(-1, C)[keep]
    else:
        p = preds.flatten()[keep]
    return p, target.flatten()[keep], True


def expect_flag(flag, bad):
    bits = int(flag.item())
    assert bits == (_native.FLAG_TARGET_RANGE if bad else 0), bits
    flag.zero_()


def check_confmat(preds, target, C, ignore_index, path):
    assert path_of("confmat", preds, target, C) == path, (preds.dtype, tuple(preds.shape), C)
    p, t, bad = admitted(preds, target, C, ignore_index)
    want = om.confusion_matrix(p, t, C, ignore_index)
    cm = torch.zeros(C, C, dtype=torch.int64, device=DEV)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    for k in (1, 2):
        _native.multiclass_confmat_update_(cm, preds, target, C, ignore_index, flag)
        expect_flag(flag, bad)
        assert torch.equal(cm, k * want), (path, preds.dtype, C, ignore_index, k, int((cm - k * want).abs().sum()))


def stats_state(C, micro):
    return [torch.zeros(1 if micro else C, dtype=torch.int64, device=DEV) for _ in range(4)], \
        torch.zeros(3 * C + 2, dtype=torch.int64, device=DEV)


def check_stats(preds, target, C, ignore_index, micro, path):
    assert path_of("stats", preds, target, C, micro) == path, (preds.dtype, tuple(preds.shape), C, micro)
    p, t, bad = admitted(preds, target, C, ignore_index)
    want = om.stat_scores(p, t, C, 1, "micro" if micro else "none", "global", ignore_index)
    want = want.reshape(4, -1)
    states, ws = stats_state(C, micro)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    for k in (1, 2):
        _native.multiclass_stat_scores_update_(*states, ws, preds, target, C, ignore_index, micro, flag)
        expect_flag(flag, bad)
        assert not bool(ws.any()), (path, "workspace left dirty", k)
        got = torch.stack(states)
        assert torch.equal(got, k * want), (path, preds.dtype, C, ignore_index, micro, k,
                                            (got - k * want).abs().sum(-1).tolist())


def check_topk(preds, target, C, k, ignore_index):
    assert path_of("topk", preds, target, C) == ("topk", "stats_global")
    p, t, bad = admitted(preds, target, C, ignore_index)
    want = om.stat_scores_topk(p, t, C, k, ignore_index)
    states, ws = stats_state(C, False)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    for rep in (1, 2):
        _native.multiclass_stat_scores_topk_update_(*states, ws, preds, target, C, k, ignore_index, flag)
        expect_flag(flag, bad)
        assert not bool(ws.any()), ("topk", "workspace left dirty", rep)
        got = torch.stack(states)
        assert torch.equal(got, rep * want), ("topk", preds.dtype, C, k, ignore_index, (got - rep * want).abs().sum(-1).tolist())


def check_samplewise(preds, target, C, ignore_index):
    """Per-sample counts over the trailing dimensions (one sample per row of a `[N, C]` input)."""
    path = path_of("samplewise", preds, target, C)
    want = om.stat_scores(preds, target, C, 1, "none", "samplewise", ignore_index)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    got = torch.stack(_native.multiclass_stat_scores_samplewise(preds, target, C, ignore_index, flag))
    expect_flag(flag, False)
    assert torch.equal(got, want), (path, preds.dtype, C, ignore_index, (got - want).abs().sum((-1, -2)).tolist())
    return path


def check_argmax(preds):
    path = path_of("argmax", preds, preds[:, 0], preds.shape[1])
    got = _native.argmax_rows(preds)
    want = preds.argmax(1)
    assert torch.equal(got, want), (path, preds.dtype, tuple(preds.shape), (got != want).nonzero()[:5].tolist())
    return path


# ------------------------------------------------------------------------------------------------------------------
# launch paths x sizes
# ------------------------------------------------------------------------------------------------------------------
def row_kernel(x) -> str:
    C = x.shape[1]
    if C < 32:
        return "strided"
    if x.element_size() > 4 or (C * x.element_size()) % 16 or x.data_ptr() % 16:
        return "scalar"
    return "vec"


@pytest.mark.parametrize("dtype", FLOATS + [torch.float64], ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("C", SIZES)
def test_row_paths_and_sizes(C, dtype):
    """Every class count of the boundary set, on the vec / scalar / strided kernels and every sink they reach, with N on
    both sides of the shared-memory switches (N = 4095 / 4096 for C <= 65, N = 4096 above)."""
    ns = (4095, 4096) if C <= 65 else (4096,) if C <= 1025 else (1500,)
    for n in ns:
        x = rows(n, C, dtype, seed=n)
        base = row_kernel(x)
        for ign in (None, -1, 0, C - 1, C):
            t = targets(n, C, torch.int64, ign, seed=C + n)
            cm_sink = "confmat_smem" if C * C <= 4096 and n >= 4096 else "confmat_global"
            check_confmat(x, t, C, ign, (base, cm_sink))
            st_sink = "stats_smem" if C <= 256 and n >= 4096 else "stats_global"
            check_stats(x, t, C, ign, False, ("vec_plain" if base == "vec" else base, st_sink))
        t = targets(n, C, torch.int64, -1, seed=C)
        check_stats(x, t, C, -1, True, ("vec_plain" if base == "vec" else base, "stats_global"))
        check_stats(x, t, C, None if C > 1 else -1, True, ("vec_plain" if base == "vec" else base, "stats_global"))
        assert check_argmax(x) == ("vec_plain" if base == "vec" else base, "argmax")
        if n == ns[-1]:
            for ign in (None, C - 1):
                ts = targets(n, C, torch.int64, ign, seed=3)
                assert check_samplewise(x, ts, C, ign) == ("vec_plain" if base == "vec" else base, "samplewise")
            for k in sorted({2, 5, C} & set(range(2, C + 1))):
                check_topk(x, targets(n, C, torch.int64, -1, seed=k), C, k, -1)
            check_topk(x, targets(n, C, torch.int64, None, seed=4), C, 1, None)


@pytest.mark.parametrize("dtype", FLOATS, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("C", [32, 64, 65, 256, 512, 1000, 1024, 2048, 4100])
def test_misaligned_base_takes_the_scalar_path(C, dtype):
    """A contiguous view whose base is not 16-byte aligned: scalar path for any C."""
    n = 4096
    x = misaligned(rows(n, C, dtype, seed=5))
    for ign in (None, -1, C - 1):
        t = targets(n, C, torch.int64, ign, seed=6)
        check_confmat(x, t, C, ign, ("scalar", "confmat_smem" if C * C <= 4096 else "confmat_global"))
        big = n * C >= 1 << 24  # the deferred fold behind the scalar kernel (no programmatic launch of its own)
        check_stats(x, t, C, ign, False, ("scalar", "stats_smem" if C <= 256 else "stats_deferred" if big else "stats_global"))
        check_stats(x, t, C, ign, True, ("scalar", "stats_deferred" if big else "stats_global"))
    assert check_argmax(x) == ("scalar", "argmax")
    assert check_samplewise(x, targets(n, C, seed=7), C, None) == ("scalar", "samplewise")


@pytest.mark.parametrize("dtype", FLOATS + [torch.float64], ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("C,d", [(2, 9), (3, 5), (31, 4), (32, 3), (257, 2), (1000, 3)])
def test_strided_class_dimension(C, d, dtype):
    """`[N, C, d1, d2]` inputs: thread per position, the class dimension strided by the trailing size."""
    n = max(2, 8192 // (C * d) + 1)
    x = rows(n * d * 2, C, dtype, seed=8).reshape(n, d, 2, C).permute(0, 3, 1, 2).contiguous()
    for ign in (None, -1, 0, C):
        t = targets(n * d * 2, C, torch.int64, ign, seed=9).reshape(n, d, 2)
        total = n * d * 2
        check_confmat(x, t, C, ign, ("strided", "confmat_smem" if C * C <= 4096 and total >= 4096 else "confmat_global"))
        check_stats(x, t, C, ign, False, ("strided", "stats_smem" if C <= 256 and total >= 4096 else "stats_global"))
        check_stats(x, t, C, ign, True, ("strided", "stats_global"))
    t = targets(n * d * 2, C, seed=10).reshape(n, d, 2)
    assert check_samplewise(x, t, C, C - 1) == ("strided", "samplewise")
    assert check_argmax(x) == ("strided", "argmax")


@pytest.mark.parametrize("pred_dtype", LABEL_DTYPES + [torch.bool], ids=lambda d: str(d)[6:])
def test_integer_label_predictions(pred_dtype):
    C = 2 if pred_dtype == torch.bool else 100
    for n, shape in ((4095, (4095,)), (4096, (4096,)), (6000, (1000, 6))):
        p = targets(n, C, pred_dtype, None, seed=11).reshape(shape)
        for tdt in (torch.int64, torch.uint8):
            for ign in ((None, -1, 0, C) if tdt == torch.int64 else (None, 0, 257)):
                t = targets(n, C, tdt, ign, seed=12).reshape(shape)
                check_confmat(p, t, C, ign, ("labels", "confmat_smem" if C * C <= 4096 and n >= 4096 else "confmat_global"))
                check_stats(p, t, C, ign, False, ("labels", "stats_smem" if n >= 4096 else "stats_global"))
                check_stats(p, t, C, ign, True, ("labels", "stats_global"))
        if len(shape) == 2:
            assert check_samplewise(p, targets(n, C, seed=13).reshape(shape), C, None) == ("labels", "samplewise")


# ------------------------------------------------------------------------------------------------------------------
# target dtypes and ignore_index in the target's dtype
# ------------------------------------------------------------------------------------------------------------------
WRAPPED = [(torch.uint8, 257), (torch.uint8, -100), (torch.uint8, -1), (torch.int8, 255), (torch.int16, 65535)]


@pytest.mark.parametrize("tdtype", LABEL_DTYPES, ids=lambda d: str(d)[6:])
def test_target_dtypes_on_the_float_paths(tdtype):
    """int8 / uint8 / int16 / int32 / int64 targets (the non-int64 instantiation with `load_label`) on vec, scalar and
    strided score paths, every sink, `ignore_index` None / -1 / 0 / C - 1 / C."""
    for dtype in FLOATS:
        for label, x in (("vec", rows(4096, 120, dtype, seed=14)),
                         ("scalar", misaligned(rows(4096, 100, dtype, seed=15))),
                         ("strided", rows(4096, 100, dtype, seed=16).reshape(2048, 2, 100).transpose(1, 2).contiguous())):
            c = x.shape[1]
            tshape = (x.shape[0],) + tuple(x.shape[2:])
            n = x.numel() // c
            for ign in (None, -1, 0, c - 1, c):
                if ign == -1 and not tdtype.is_signed:
                    continue
                t = targets(n, c, tdtype, ign, seed=17).reshape(tshape)
                check_confmat(x, t, c, ign, (label, "confmat_global"))
                check_stats(x, t, c, ign, False, (label if label != "vec" else "vec_plain", "stats_smem"))
                check_stats(x, t, c, ign, True, (label if label != "vec" else "vec_plain", "stats_global"))
            if label != "strided":
                check_topk(x, targets(n, c, tdtype, None, seed=18), c, 3, None)
                check_topk(x, targets(n, c, tdtype, c, seed=18), c, 3, c)


@pytest.mark.parametrize("tdtype,ign", WRAPPED, ids=[f"{str(d)[6:]}-{i}" for d, i in WRAPPED])
def test_ignore_index_is_compared_in_the_target_dtype(tdtype, ign):
    """uint8 257 drops class 1, -100 drops 156 and -1 drops 255; int8 255 and int16 65535 drop -1.  The rows holding the
    wrapped value are ignored, not counted (in range) and not flagged (out of range)."""
    C = 10
    w = stored(ign, tdtype)
    for dtype in FLOATS:
        x = rows(8192, C, dtype, seed=19)
        xv = rows(8192, 32, dtype, seed=20)
        for xx, c in ((x, C), (xv, 32)):
            t = targets(xx.shape[0], c, tdtype, None, seed=21)
            t[::5] = w
            assert bool((t == ign).any()) and int((t == ign).sum()) == int((t == w).sum())
            k = row_kernel(xx)
            check_confmat(xx, t, c, ign, (k, "confmat_global" if c * c > 4096 else "confmat_smem"))
            check_stats(xx, t, c, ign, False, ("vec_plain" if k == "vec" else k, "stats_smem"))
            check_stats(xx, t, c, ign, True, ("vec_plain" if k == "vec" else k, "stats_global"))
            check_topk(xx, t, c, 2, ign)
            check_samplewise(xx, t, c, ign)
            check_confmat(t.to(torch.int64).clamp(0, c - 1), t, c, ign, ("labels", "confmat_smem" if c * c <= 4096 else "confmat_global"))


def test_wrapped_ignore_index_through_the_functionals():
    """The public functionals with validate_args=True: uint8 targets holding 255 with ignore_index=-1 are valid input (the
    reference ignores them and does not raise), and ignore_index=257 drops class 1."""
    import metrics_b200.functional.classification as fc

    C = 5
    x = rows(4096, C, torch.float32, seed=22)
    t = targets(4096, C, torch.uint8, None, seed=23)
    t[::7] = 255
    want = om.confusion_matrix(x, t, C, -1)
    assert torch.equal(fc.multiclass_confusion_matrix(x, t, C, ignore_index=-1), want)
    s = om.stat_scores(x, t, C, 1, "none", "global", -1)
    got = fc.multiclass_stat_scores(x, t, C, average="none", ignore_index=-1)
    assert torch.equal(got[:, :4].T, s)
    t2 = targets(4096, C, torch.uint8, None, seed=24)
    assert torch.equal(fc.multiclass_confusion_matrix(x, t2, C, ignore_index=257), om.confusion_matrix(x, t2, C, 257))
    assert int(fc.multiclass_confusion_matrix(x, t2, C, ignore_index=257)[1].sum()) == 0


# ------------------------------------------------------------------------------------------------------------------
# row contents: every half-precision bit pattern as a row maximum
# ------------------------------------------------------------------------------------------------------------------
def every_pattern_rows(dtype, C: int) -> torch.Tensor:
    """65 536 rows; row i's maximum is bit pattern i (a NaN, +-inf, a subnormal, -0 ...), at a random column and, in a third
    of the rows, again at a later column.  The other scores are random values below it (-inf where none is)."""
    g = torch.Generator().manual_seed(25)
    pat = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(dtype).to(torch.float64)
    bg = torch.randn(65536, C, generator=g, dtype=torch.float64) * pat.abs().clamp(1, 1e4).nan_to_num(1)[:, None]
    bg = bg.to(dtype).to(torch.float64)
    bg = torch.where(bg >= pat[:, None], torch.tensor(float("-inf"), dtype=torch.float64), bg)
    j = torch.randint(0, C, (65536,), generator=g)
    r = torch.arange(65536)
    bg[r, j] = pat
    dup = (r % 3 == 0)
    bg[r[dup], (j[dup] + 1 + r[dup] % (2 * chunk_cols(dtype))).clamp(max=C - 1)] = pat[dup]
    y = bg.to(dtype)
    y.view(torch.int16)[r, j] = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)  # NaN payloads exact
    return y.to(DEV)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=lambda d: str(d)[6:])
def test_every_half_precision_pattern_as_a_row_maximum(dtype):
    C = 1032  # two chunks, the second one a single (clamp-duplicated) vector
    x = every_pattern_rows(dtype, C)
    t = targets(65536, C, torch.int64, -1, seed=26)
    assert check_argmax(x) == ("vec_plain", "argmax")
    check_confmat(x, t, C, -1, ("vec", "confmat_global"))
    check_stats(x, t, C, -1, False, ("vec", "stats_deferred"))
    check_stats(x[:4096], t[:4096], C, -1, False, ("vec_plain", "stats_global"))
    xs = misaligned(x)
    assert check_argmax(xs) == ("scalar", "argmax")
    check_confmat(xs, t, C, -1, ("scalar", "confmat_global"))
    xn = x[:, :1000].reshape(8192, 8, 1000).transpose(1, 2).contiguous()
    assert check_argmax(xn) == ("strided", "argmax")
    check_confmat(xn, t.reshape(8192, 8).clamp(max=999), 1000, -1, ("strided", "confmat_global"))
    check_topk(x[:4096], t[:4096], C, 2, -1)


# ------------------------------------------------------------------------------------------------------------------
# error word, deferred fold, many chunks, large inputs
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("where", ["first", "last", "tail"])
def test_error_word_on_out_of_range_targets(where):
    """A target outside [0, C) that is not ignored sets the error word and is skipped, on each kernel; the other rows are
    counted as the chain counts them."""
    for x, C, ksink in ((rows(4096, 64, torch.bfloat16, seed=27), 64, "vec"), (rows(4099, 33, torch.float32, seed=28), 33, "scalar"),
                        (rows(4096, 7, torch.float16, seed=29), 7, "strided")):
        n = x.shape[0]
        r = {"first": 0, "last": n - 1, "tail": n - 1 - (n % 8 or 5)}[where]
        for tdt, ign in ((torch.int64, None), (torch.int64, -1), (torch.int64, C), (torch.uint8, 257), (torch.int8, 255)):
            t = targets(n, C, tdt, ign, seed=30, bad=(r,))
            k = row_kernel(x)
            check_confmat(x, t, C, ign, (k, "confmat_smem" if C * C <= 4096 and n >= 4096 else "confmat_global"))
            check_stats(x, t, C, ign, False, ("vec_plain" if k == "vec" else k, "stats_smem"))
            check_stats(x, t, C, ign, True, ("vec_plain" if k == "vec" else k, "stats_global"))
            if k != "strided":
                check_topk(x, t, C, 2, ign)
        lab = targets(4096, 50, torch.int32, None, seed=31)
        t = targets(4096, 50, torch.int64, None, seed=32, bad=({"first": 0, "last": 4095, "tail": 4093}[where],))
        check_confmat(lab, t, 50, None, ("labels", "confmat_smem"))


@pytest.mark.parametrize("dtype", FLOATS, ids=lambda d: str(d)[6:])
def test_deferred_fold(dtype):
    """N * C >= 2^24: the row kernel only REDs into the workspace and a one-CTA kernel folds; micro and macro, with
    ignore_index, chunk-edge rows and a misaligned-size tail."""
    C = 1024
    n = (1 << 24) // C + 7
    x = rows(n, C, dtype, seed=33)
    for ign in (None, -1, 0, C - 1, C):
        t = targets(n, C, torch.int64, ign, seed=34)
        check_stats(x, t, C, ign, False, ("vec", "stats_deferred"))
        check_stats(x, t, C, ign, True, ("vec", "stats_deferred"))
    t = targets(n, C, torch.int16, 65535, seed=35)
    check_stats(x, t, C, 65535, False, ("vec", "stats_deferred"))
    xs = x[: (1 << 24) // C - 1]  # one row short of the switch: the single launch with the last-CTA fold
    check_stats(xs, targets(xs.shape[0], C, seed=36), C, None, False, ("vec_plain", "stats_global"))


def test_many_chunks():
    """C = 70 000 (69 chunks of bfloat16): the chunk loop and the deferred fold over a large state.  The chain's C^2
    bincount does not fit in memory, so the macro counts are its diag / column / row sums taken with C-length bincounts."""
    C, n = 70000, 256
    x = rows(n, C, torch.bfloat16, seed=37)
    t = targets(n, C, torch.int64, -1, seed=38)
    check_stats(x, t, C, -1, True, ("vec", "stats_deferred"))
    keep = t != -1
    p, tt = x.argmax(1)[keep], t[keep]
    tp = torch.bincount(tt[p == tt], minlength=C)
    fp = torch.bincount(p, minlength=C) - tp
    fn = torch.bincount(tt, minlength=C) - tp
    want = torch.stack([tp, fp, keep.sum() - (tp + fp + fn), fn])
    states, ws = stats_state(C, False)
    assert path_of("stats", x, t, C) == ("vec", "stats_deferred")
    for k in (1, 2):
        _native.multiclass_stat_scores_update_(*states, ws, x, t, C, -1, False)
        assert not bool(ws.any())
        assert torch.equal(torch.stack(states), k * want), k
    assert check_argmax(x) == ("vec_plain", "argmax")


def test_more_than_2_31_scores():
    """`[2^21 + 3, 1024]` bfloat16 (about 4.3 GB): row offsets past 2^31 elements, confusion matrix and deferred stats;
    the chain runs in row chunks and its counts add up."""
    n, C = (1 << 21) + 3, 1024
    need = n * C * 2 + (3 << 30)
    if torch.cuda.mem_get_info(DEV)[0] < need:
        pytest.skip(f"needs {need >> 30} GiB of free device memory")
    g = torch.Generator(device=DEV).manual_seed(39)
    x = torch.randn(n, C, generator=g, device=DEV, dtype=torch.bfloat16)
    tail = rows(4096, C, torch.bfloat16, seed=40)
    x[-4096:] = tail  # the row kinds where the offsets exceed 2^31
    t = torch.randint(-1, C, (n,), generator=g, device=DEV)
    assert x.numel() > 2**31
    cm = torch.zeros(C, C, dtype=torch.int64, device=DEV)
    states, ws = stats_state(C, False)
    assert path_of("confmat", x, t, C) == ("vec", "confmat_global")
    assert path_of("stats", x, t, C) == ("vec", "stats_deferred")
    _native.multiclass_confmat_update_(cm, x, t, C, -1)
    _native.multiclass_stat_scores_update_(*states, ws, x, t, C, -1, False)
    want_cm = torch.zeros_like(cm)
    want_st = torch.zeros(4, C, dtype=torch.int64, device=DEV)
    step = 1 << 18
    for r in range(0, n, step):
        want_cm += om.confusion_matrix(x[r: r + step], t[r: r + step], C, -1)
        want_st += om.stat_scores(x[r: r + step], t[r: r + step], C, 1, "none", "global", -1)
    assert torch.equal(cm, want_cm), int((cm - want_cm).abs().sum())
    assert torch.equal(torch.stack(states), want_st)
    assert not bool(ws.any())


# ------------------------------------------------------------------------------------------------------------------
# back-to-back updates: consecutive programmatic launches into one state
# ------------------------------------------------------------------------------------------------------------------
def test_back_to_back_updates():
    """Each sink on the vec path at C = 32 / 1000 / 1024 in every score dtype, then eight distinct resident batches updated
    back to back with no host synchronisation in between: each launch waits for the previous grid of the stream."""
    for dtype in FLOATS:
        for C, n in ((32, 4096), (1000, 4096), (1024, 1200)):
            x = rows(n, C, dtype, seed=41)
            if (C * x.element_size()) % 16:
                continue
            for ign in (None, -1, C - 1):
                t = targets(n, C, torch.int64, ign, seed=42)
                check_confmat(x, t, C, ign, path_of("confmat", x, t, C))
                check_stats(x, t, C, ign, False, path_of("stats", x, t, C))
                check_stats(x, t, C, ign, True, path_of("stats", x, t, C, True))
            check_argmax(x)
            check_samplewise(x, targets(n, C, seed=43), C, None)
    C, n = 1000, (1 << 24) // 1000 + 5
    xs = [rows(n, C, torch.bfloat16, seed=44 + i) for i in range(8)]
    ts = [targets(n, C, torch.int64, -1, seed=60 + i) for i in range(8)]
    cm_path = path_of("confmat", xs[0], ts[0], C)
    st_path = path_of("stats", xs[0], ts[0], C)
    assert cm_path == ("vec", "confmat_global")
    assert st_path == ("vec", "stats_deferred")
    cm = torch.zeros(C, C, dtype=torch.int64, device=DEV)
    states, ws = stats_state(C, False)
    for x, t in zip(xs, ts):  # back to back, no host synchronisation in between
        _native.multiclass_confmat_update_(cm, x, t, C, -1)
        _native.multiclass_stat_scores_update_(*states, ws, x, t, C, -1, False)
    want_cm = sum(om.confusion_matrix(x, t, C, -1) for x, t in zip(xs, ts))
    want_st = sum(om.stat_scores(x, t, C, 1, "none", "global", -1) for x, t in zip(xs, ts))
    assert torch.equal(cm, want_cm), (cm_path, int((cm - want_cm).abs().sum()))
    assert torch.equal(torch.stack(states), want_st), st_path
    assert not bool(ws.any())
    cm.zero_()
    for x, t in zip(xs, ts):
        _native.multiclass_confmat_update_(cm, x, t, C, -1)
    assert torch.equal(cm, want_cm), "confusion matrix alone, back to back"


# ------------------------------------------------------------------------------------------------------------------
# entry points: the functionals and the torch.ops binding
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_binding():
    from metrics_b200 import torch_ops

    torch_ops.load()
    return torch.ops.metrics_b200


@pytest.mark.parametrize("tdtype,ign", [(torch.int64, None), (torch.int64, -1), (torch.int16, 0)] + WRAPPED,
                         ids=lambda v: str(v)[6:] if isinstance(v, torch.dtype) else str(v))
def test_entry_points(tdtype, ign, torch_binding, monkeypatch):
    """The functionals (validate_args on and off) and the `torch.ops.metrics_b200` binding count what the chain counts."""
    import metrics_b200.functional.classification as fc

    C = 10
    for dtype in FLOATS:
        for x in (rows(4096, C, dtype, seed=70), rows(4096, 64, dtype, seed=71), misaligned(rows(512, 64, dtype, seed=72))):
            c, n = x.shape[1], x.shape[0]
            t = targets(n, c, tdtype, ign, seed=73)
            if ign is not None and stored(ign, tdtype) != ign:
                t[::6] = stored(ign, tdtype)
            cm = om.confusion_matrix(x, t, c, ign)
            st = om.stat_scores(x, t, c, 1, "none", "global", ign)
            mi = om.stat_scores(x, t, c, 1, "micro", "global", ign)
            for validate in (True, False):
                assert torch.equal(fc.multiclass_confusion_matrix(x, t, c, ignore_index=ign, validate_args=validate), cm)
                got = fc.multiclass_stat_scores(x, t, c, average="none", ignore_index=ign, validate_args=validate)
                assert torch.equal(got[:, :4].T, st)
                got = fc.multiclass_stat_scores(x, t, c, average="micro", ignore_index=ign, validate_args=validate)
                assert torch.equal(got[:4], mi)
                got = fc.multiclass_stat_scores(x, t, c, average="none", top_k=2, ignore_index=ign, validate_args=validate)
                assert torch.equal(got[:, :4].T, om.stat_scores_topk(x, t, c, 2, ign))
            x3, t3 = x[: n - n % 8].reshape(-1, 8, c).transpose(1, 2), t[: n - n % 8].reshape(-1, 8)
            got = fc.multiclass_stat_scores(x3, t3, c, average="none", multidim_average="samplewise", ignore_index=ign)
            assert torch.equal(got[..., :4].permute(2, 0, 1), om.stat_scores(x3, t3, c, 1, "none", "samplewise", ign))
            # the operator binding, directly and behind the ctypes wrappers' switch
            b = torch.zeros(c, c, dtype=torch.int64, device=DEV)
            torch_binding.confmat_update_(b, x, t, c, ign)
            assert torch.equal(b, cm)
            sb = [torch.zeros(c, dtype=torch.int64, device=DEV) for _ in range(4)]
            ws = torch.zeros(3 * c + 2, dtype=torch.int64, device=DEV)
            torch_binding.stat_scores_update_(*sb, ws, x, t, c, ign)
            assert torch.equal(torch.stack(sb), st) and not bool(ws.any())
            with monkeypatch.context() as m:
                m.setattr(_native, "_TORCH_BINDING", True)
                check_confmat(x, t, c, ign, path_of("confmat", x, t, c))
                check_stats(x, t, c, ign, False, path_of("stats", x, t, c))
                check_stats(x, t, c, ign, True, path_of("stats", x, t, c, True))
