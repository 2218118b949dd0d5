"""GPU: kernel K4 (`mb200_binned_curve_update[_multilabel]`, csrc/binned.cu) against the reference's own binned-state chain
(oracle/binned_counts.py) run on the same GPU, bit for bit (`torch.equal` on the int64 `[T, (C,) 2, 2]` state), on every
launch path of `binned_update_impl`:
  fast     binary, float32 scores, 16-byte aligned, n in [4096, 2^31), T <= 2048: int64 / int32 / uint8 / bool / int8 labels
           with n a multiple of 8, of 4 only, and neither (scalar tail), and n = 4095 / 4096 on either side of the minimum
  generic  counters in shared memory / global atomics (C * 2 * (T + 1) * 4 bytes on either side of 40 KB), comparands in
           shared memory / global memory (T = 2048 / 2049, and float64 comparands beside large counters), misaligned views,
           binary, multiclass and multilabel, 32- and 64-bit indices (n * C >= 2^31)
Every case asserts its path with `path_of`, which restates the dispatch.  The comparison is the reference's: on its loop
branch (binary n > 50 000, multiclass n * C * C > 10^6) in the score dtype, else in the promoted dtype, so every score dtype
meets every threshold dtype on both sides of both size rules.  Each case runs the ctypes binding once and the `torch.ops`
binding twice into one state (which must then hold twice the chain) and checks that the scratch words, ticket included, are
zero after each call.  The edge cases hold thresholds at +-0, subnormals, 1.0, NaN, +-inf and values the score dtype cannot
represent; scores on each threshold, on its rounding and on the neighbours of that; and every float16 / bfloat16 bit pattern.
"""
import importlib

import pytest
import torch

from metrics_b200 import _native, torch_ops
from oracle import binned_counts as ob

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F16, BF16, F32, F64 = torch.float16, torch.bfloat16, torch.float32, torch.float64
SCORES = [F16, BF16, F32, F64]
THR_DTYPES = [F16, BF16, F32, F64, torch.int64]
FAST_LABELS = [torch.int64, torch.int32, torch.uint8, torch.bool, torch.int8]
# unsorted, duplicated, not representable in half precision or float32, +-0, subnormal
THR_VALUES = [0.5, 0.1, 0.9999, 0.3, 0.0, 1.0, 0.3, 0.7, 0.33333333, 0.9, 0.2, 1e-40, -0.0, 0.70000001]
EDGE_THR = THR_VALUES + [float("nan"), float("inf"), float("-inf"), 6e-8, 1e-45, -1e-40, 65504.0, 1e300]


# ------------------------------------------------------------------------------------------------------------------
# the dispatch of binned.cu, restated
# ------------------------------------------------------------------------------------------------------------------
def _aligned(t):
    return t.data_ptr() % 16 == 0


def path_of(preds, target, num_classes, num_thresholds, multilabel=False):
    n = preds.shape[0] if multilabel else target.numel()
    C, T = num_classes, num_thresholds
    if (not multilabel and C == 1 and preds.dtype == F32 and target.dtype in FAST_LABELS and T <= 2048 and n < 2**31
            and n >= 4096 and _aligned(preds) and _aligned(target)):
        return ("fast",)
    counters = C * 2 * (T + 1) * 4
    smem = counters <= 40 * 1024
    comparand = 8 if preds.dtype == F64 else 4
    thr_smem = T <= 2048 and (counters if smem else 0) + T * comparand <= 48 * 1024
    return ("generic", "smem" if smem else "global", "thr_smem" if thr_smem else "thr_global",
            "idx64" if n * C >= 2**31 else "idx32")


def thresholds(dtype, values=THR_VALUES):
    if dtype == torch.int64:
        return torch.tensor([1, 0, 0, 2, -1], dtype=torch.int64, device=DEV)
    return torch.tensor(values, dtype=F64, device=DEV).to(dtype)


def oracle(preds, target, num_classes, thr, multilabel=False, ignore_index=None):
    """The reference's update on a formatted batch (scores already probabilities)."""
    if multilabel:
        return ob.multilabel(preds, target, num_classes, thr, ignore_index)
    if num_classes == 1:
        return ob.binary_update(preds, target, thr)
    return ob.multiclass_update(preds, target, num_classes, thr)


def check(preds, target, thr, num_classes=1, want_path=None, multilabel=False, ignore_index=None, want=None):
    """ctypes once, torch.ops twice into one state; scratch zero after each call; both equal to the chain."""
    T = thr.numel()
    if want_path is not None:
        assert path_of(preds, target, num_classes, T, multilabel) == want_path
    if want is None:
        want = oracle(preds, target, num_classes, thr, multilabel, ignore_index)
    got = _native.binned_curve_update(preds, target, thr, num_classes, multilabel=multilabel, ignore_index=ignore_index)
    info = (want_path, preds.dtype, thr.dtype, tuple(preds.shape), target.dtype, ignore_index)
    assert torch.equal(got, want), info
    ops = torch_ops.ops()
    srt, order = torch.sort(thr)
    state = torch.zeros((T, num_classes, 2, 2), dtype=torch.int64, device=DEV)
    scratch = torch.zeros(int(_native.lib().mb200_binned_curve_scratch_words(num_classes, T)), dtype=torch.int64, device=DEV)
    for k in (1, 2):
        ops.binned_curve_update_(state, scratch, preds, target, srt.contiguous(), num_classes, multilabel, ignore_index)
        assert int(scratch.count_nonzero()) == 0, info
    acc = state if multilabel or num_classes > 1 else state[:, 0]
    assert torch.equal(acc, 2 * want[order]), info
    return got


@pytest.fixture(scope="module", autouse=True)
def _ops():
    torch_ops.load()


def gen(shape, dtype, seed):
    return ob.scores_near(torch.tensor(THR_VALUES, dtype=F64), shape, dtype, seed).to(DEV)


def labels(shape, high, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, high, shape, generator=g).to(dtype).to(DEV)


# ------------------------------------------------------------------------------------------------------------------
# fast path
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("label_dtype", FAST_LABELS, ids=str)
@pytest.mark.parametrize("n", [4095, 4096, 8192, 8196, 8195, 50_000, 50_001])
def test_binary_fast_path_labels_and_tails(label_dtype, n):
    p = gen((n,), F32, n)
    t = labels((n,), 2, label_dtype, n + 1)
    for thr in (thresholds(F32), thresholds(F64), torch.linspace(0, 1, 200, device=DEV)):
        check(p, t, thr, want_path=("fast",) if n >= 4096 else ("generic", "smem", "thr_smem", "idx32"))


def test_binary_fast_path_misaligned_view_takes_the_generic_kernel():
    p, t = gen((8193,), F32, 7), labels((8193,), 2, torch.int64, 8)
    check(p[1:], t[1:], thresholds(F64), want_path=("generic", "smem", "thr_smem", "idx32"))
    check(p[1:], t[1:].clone(), thresholds(F32), want_path=("generic", "smem", "thr_smem", "idx32"))


# ------------------------------------------------------------------------------------------------------------------
# generic kernel: every score dtype x threshold dtype on both sides of both size rules
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("score", SCORES, ids=str)
@pytest.mark.parametrize("thr_dtype", THR_DTYPES, ids=str)
@pytest.mark.parametrize("n", [50_000, 50_001])
def test_binary_branches(score, thr_dtype, n):
    p = gen((n,), score, n + 17)
    t = labels((n,), 2, torch.int32, n)
    path = ("fast",) if score == F32 else ("generic", "smem", "thr_smem", "idx32")
    check(p, t, thresholds(thr_dtype), want_path=path)


@pytest.mark.parametrize("score", SCORES, ids=str)
@pytest.mark.parametrize("thr_dtype", THR_DTYPES, ids=str)
@pytest.mark.parametrize("n", [10_000, 10_001])
def test_multiclass_branches(score, thr_dtype, n):
    C = 10
    p, t = gen((n, C), score, n + 31), labels((n,), C, torch.int64, n)
    check(p, t, thresholds(thr_dtype), C, want_path=("generic", "smem", "thr_smem", "idx32"))


@pytest.mark.parametrize("C, path", [(25, ("generic", "smem", "thr_smem", "idx32")), (26, ("generic", "global", "thr_smem", "idx32"))])
@pytest.mark.parametrize("score", [F16, F32], ids=str)
def test_counters_in_shared_and_global_memory(C, path, score):
    thr = torch.linspace(0, 1, 200, device=DEV, dtype=F64)
    for n in (1000, 1700):  # N * C * C on either side of 10^6
        check(gen((n, C), score, C + n), labels((n,), C, torch.int64, n), thr, C, want_path=path)


@pytest.mark.parametrize("T", [2048, 2049])
@pytest.mark.parametrize("score", SCORES, ids=str)
def test_thresholds_in_shared_and_global_memory(T, score):
    thr = torch.rand(T, generator=torch.Generator().manual_seed(T), dtype=F64).to(DEV)
    n = 60_000
    p, t = gen((n,), score, T), labels((n,), 2, torch.int16, T)
    want = ("generic", "smem", "thr_smem" if T <= 2048 else "thr_global", "idx32")  # 2 * (T + 1) counters: shared memory
    check(p, t, thr, want_path=want)  # int16 labels: never the fast path
    if score == F32 and T <= 2048:
        want = ("fast",)
    check(p[:40_000], labels((40_000,), 2, torch.int64, T), thr.to(F32), want_path=want)


def test_float64_comparands_beside_large_counters_stay_in_global_memory():
    C, T = 4, 1250  # 40 032 bytes of counters: float comparands fit beside them, double ones do not
    thr = torch.rand(T, generator=torch.Generator().manual_seed(5), dtype=F64).to(DEV)
    for score, path in ((F64, ("generic", "smem", "thr_global", "idx32")), (F32, ("generic", "smem", "thr_smem", "idx32"))):
        for n in (1000, 70_000):
            check(gen((n, C), score, n), labels((n,), C, torch.int64, n), thr, C, want_path=path)


def test_misaligned_multiclass_views():
    C = 3
    p, t = gen((20_001, C), F16, 3), labels((20_001,), C, torch.int64, 3)
    flat = p.flatten()[1:1 + 20_000 * C].view(20_000, C)  # base 2 bytes past an allocation
    check(flat, t[1:], thresholds(F32), C, want_path=("generic", "smem", "thr_smem", "idx32"))


# ------------------------------------------------------------------------------------------------------------------
# multilabel: promoted dtype always, ignore_index in the target's dtype
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("score", SCORES, ids=str)
@pytest.mark.parametrize("target_dtype, ignore_index", [
    (torch.int64, None), (torch.int64, 0), (torch.int64, 1), (torch.int64, -1), (torch.uint8, 257), (torch.uint8, 0),
    (torch.uint8, 1), (torch.uint8, -1), (torch.int8, 255), (torch.int32, -100)])
def test_multilabel_ignore_index(score, target_dtype, ignore_index):
    n, L = 3000, 5
    p = gen((n, L), score, L)
    t = labels((n, L), 2, torch.int64, n)
    if ignore_index is not None and ignore_index not in (0, 1):
        wrapped = torch.tensor(ignore_index).to(target_dtype).to(torch.int64)  # what the target holds for it
        t[::4, 2] = wrapped
    t = t.to(target_dtype)
    for thr_dtype in (F16, F32, F64):
        got = check(p, t, thresholds(thr_dtype), L, want_path=("generic", "smem", "thr_smem", "idx32"), multilabel=True,
                    ignore_index=ignore_index)
        if ignore_index is not None:
            kept = int(got[0].sum())
            assert kept < n * L  # the ignored entries are not in the state
    # the functional, with validation (which accepts the wrapped value), on the same state
    prc = importlib.import_module("metrics_b200.functional.classification.precision_recall_curve")
    thr = thresholds(F64)
    got = prc.multilabel_precision_recall_curve(p, t, L, thresholds=thr, ignore_index=ignore_index)
    want = prc._multilabel_precision_recall_curve_compute(ob.multilabel(p, t, L, thr, ignore_index), L, thr)
    assert all(torch.equal(a, b) for a, b in zip(got, want))


# ------------------------------------------------------------------------------------------------------------------
# edge values
# ------------------------------------------------------------------------------------------------------------------
def _all_patterns(dtype):
    return torch.arange(-(2**15), 2**15, dtype=torch.int32).to(torch.int16).view(dtype).to(DEV)


def _near(thr, dtype):
    """Each threshold, its rounding in `dtype`, and the two neighbours of that rounding."""
    bits = {F16: torch.int16, BF16: torch.int16, F32: torch.int32, F64: torch.int64}[dtype]
    r = thr.to(F64).to(dtype)
    b = r.view(bits)
    return torch.cat([thr.to(dtype), r, (b + 1).view(dtype), (b - 1).view(dtype)])


@pytest.mark.parametrize("score", SCORES, ids=str)
@pytest.mark.parametrize("thr_dtype", [F16, BF16, F32, F64], ids=str)
def test_edge_thresholds_and_scores(score, thr_dtype):
    thr = thresholds(thr_dtype, EDGE_THR)
    base = _near(thr, score)
    if score in (F16, BF16):
        base = torch.cat([base, _all_patterns(score)])
    else:
        base = torch.cat([base, _all_patterns(F16).to(score), _all_patterns(BF16).to(score)])
    for n in (50_000, 50_001 + base.numel()):  # both branches
        g = torch.Generator().manual_seed(n)
        p = base[torch.randint(0, base.numel(), (n,), generator=g).to(DEV)]
        p[: min(n, base.numel())] = base[: min(n, base.numel())]
        t = labels((n,), 2, torch.int64, n)
        check(p, t, thr)


# ------------------------------------------------------------------------------------------------------------------
# 64-bit indices
# ------------------------------------------------------------------------------------------------------------------
def test_64bit_index_path():
    """f16 [2^30, 2]: n * C = 2^31.  The chain is the reference's loop branch run on row chunks (its counts add up), so the
    peak stays near the 5 GiB of input."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    n, C = 2**30, 2
    g = torch.Generator(device=DEV).manual_seed(3)
    p = torch.rand((n, C), generator=g, device=DEV, dtype=F16)
    t = torch.randint(0, C, (n,), generator=g, device=DEV, dtype=torch.uint8)
    thr = torch.tensor([0.3, 0.5, 0.70000001], device=DEV, dtype=F64)
    assert path_of(p, t, C, 3) == ("generic", "smem", "thr_smem", "idx64")
    want = torch.zeros((3, C, 2, 2), dtype=torch.int64, device=DEV)
    step = 2**25
    for lo in range(0, n, step):
        want += ob.multiclass_update_loop(p[lo:lo + step], t[lo:lo + step].long(), C, thr)
    got = _native.binned_curve_update(p, t, thr, C)
    assert torch.equal(got, want)
    assert torch.cuda.max_memory_allocated() < 10 * 2**30
    del p, t
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# metric classes and functionals
# ------------------------------------------------------------------------------------------------------------------
def test_metric_classes_over_batches_straddling_the_branch_boundary():
    from metrics_b200.classification import BinaryPrecisionRecallCurve, MulticlassPrecisionRecallCurve

    thr = thresholds(F64).sort().values
    m = BinaryPrecisionRecallCurve(thresholds=thr).to(DEV)
    want = 0
    for k, n in enumerate((30_000, 60_000, 50_000, 50_001)):
        p, t = gen((n,), F16, 100 + k), labels((n,), 2, torch.int64, 100 + k)
        m.update(p, t)
        want = want + ob.binary(p, t, thr)
    assert torch.equal(m.confmat, want)
    mc = MulticlassPrecisionRecallCurve(num_classes=10, thresholds=thr).to(DEV)
    want = 0
    for k, n in enumerate((5_000, 12_000)):
        p, t = gen((n, 10), BF16, 200 + k), labels((n,), 10, torch.int64, 200 + k)
        mc.update(p, t)
        want = want + ob.multiclass(p, t, 10, thr)
    assert torch.equal(mc.confmat, want)


@pytest.mark.parametrize("logits", [False, True])
@pytest.mark.parametrize("score", [F16, BF16, F32], ids=str)
def test_functionals(logits, score):
    prc = importlib.import_module("metrics_b200.functional.classification.precision_recall_curve")
    thr = thresholds(F64)
    for n in (40_000, 70_000):
        p = gen((n,), score, n)
        if logits:
            p = (p.float() * 8 - 4).to(score)
        t = labels((n,), 2, torch.int64, n)
        fp, ft, fthr = prc._binary_precision_recall_curve_format(p, t, thr, None)
        state = prc._binary_precision_recall_curve_update(fp, ft, fthr)
        assert torch.equal(state, ob.binary(p, t, thr)), (n, logits, score)
        got = prc.binary_precision_recall_curve(p, t, thresholds=thr)
        want = prc._binary_precision_recall_curve_compute(ob.binary(p, t, thr), thr)
        assert all(torch.equal(a, b) for a, b in zip(got, want))
        pm = gen((n // 10, 10), score, n + 1)
        if logits:
            pm = (pm.float() * 8 - 4).to(score)
        tm = labels((n // 10,), 10, torch.int64, n)
        for avg in (None, "micro"):
            fp, ft, fthr = prc._multiclass_precision_recall_curve_format(pm, tm, 10, thr, None, avg)
            state = prc._multiclass_precision_recall_curve_update(fp, ft, 10, fthr, avg)
            assert torch.equal(state, ob.multiclass(pm, tm, 10, thr, None, avg)), (n, logits, score, avg)
