"""GPU: kernel K2 (`mb200_binary_stat_counts*`, csrc/binary.cu) against the reference's own chain of torch ops
(oracle/binary_counts.py) run on the same GPU, on every launch path of `binary_stat_counts_impl`:

  single pass      binary, global, int64 target, 16-byte aligned, float32 / float16 / bfloat16 scores, large scratch
  two pass (flat)  the same with float64 scores, or through the 4-byte-scratch entry `mb200_binary_stat_counts`
  column owner     `[N, L]` multilabel, global, 2 <= L <= 256
  generic, shared  every other float shape with at most 2048 groups
  generic, global  more than 2048 groups
  labels           integer predictions (shared or global groups)

and on the generic kernel's 64-bit index arithmetic (2^31 elements and more).  The counts are int64 and compared exactly.

The scores are where threshold comparisons go wrong: all 65 536 float16 / bfloat16 bit patterns (as logits, and the ones
in [0, 1] as probabilities with and without NaN), and for float32 / float64 the 64 neighbours on each side of the
threshold rounded to the dtype and of logit(threshold).  The thresholds are mostly not representable in half precision:
the reference compares `preds > threshold` after ATen has rounded the Python float to the score dtype, so a bfloat16
score of 0.30078125 is not above 0.3.  Every case first asserts which path the kernel takes (`path_of` restates the
dispatch), so a change to the dispatch shows up as a failure rather than as a path that quietly stops being tested.
"""
import ctypes
import math

import pytest
import torch

from metrics_b200 import _native
from oracle import binary_counts as ob

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HALF = (torch.float16, torch.bfloat16)
DTYPES = [torch.float32, torch.float16, torch.bfloat16, torch.float64]
THRESHOLDS = [0.5, 0.3, 0.1, 1 / 3, 0.7, 0.9, 0.999, 0.9999, 1e-4, 0.0, 1.0,
              # ATen rounds the scalar to float32 first, then to half precision: these land on the other side of a
              # half-precision midpoint than one direct rounding would
              0.5 + 2**-12 + 2**-40, 0.5 + 2**-9 + 2**-40]
F16_SUBNORMAL = [2e-6, 6e-6, 1.2e-5, 3e-5, 6e-5]  # thr * 2^-9 is below float16's absolute spacing (2^-24) there
CASES = [(d, t) for d in DTYPES for t in THRESHOLDS] + [(torch.float16, t) for t in F16_SUBNORMAL]
CASE_IDS = [f"{str(d)[6:]}-{t:.6g}" for d, t in CASES]
KINDS = {torch.float16: ("logits", "probs", "probs_nan"), torch.bfloat16: ("logits", "probs", "probs_nan")}
SMEM_GROUPS = 2048  # binary.cu: groups privatised in shared memory up to this many


def path_of(preds, target, num_labels, samplewise, large_scratch=True):
    """(launch path, 32-bit index arithmetic) that `binary_stat_counts_impl` takes for these arguments."""
    n_outer = preds.shape[0]
    total = preds.numel()
    inner = total // (n_outer * num_labels)
    groups = n_outer * num_labels if samplewise else num_labels
    floating = preds.is_floating_point()
    aligned = (preds.data_ptr() | target.data_ptr()) % 16 == 0
    flat = floating and not samplewise and num_labels == 1 and target.dtype == torch.int64 and aligned
    if flat and preds.dtype != torch.float64 and large_scratch:
        path = "single_pass"
    elif flat:
        path = "two_pass"
    elif floating and not samplewise and inner == 1 and 2 <= num_labels <= 256:
        path = "columns"
    else:
        path = ("generic" if floating else "labels") + ("_shared" if groups <= SMEM_GROUPS else "_global")
    return path, total < 2**31


def kernel(preds, target, num_labels, threshold, ignore_index, samplewise, err_flag=None):
    """The default wrapper (large scratch: the single pass where it applies)."""
    return _native.binary_stat_counts(preds, target, num_labels, threshold, ignore_index, samplewise, None, err_flag)


def two_pass(preds, target, num_labels, threshold, ignore_index, samplewise):
    """The 4-byte-scratch entry: the vote pass, then the counting kernel."""
    n_outer = preds.shape[0]
    inner = preds.numel() // (n_outer * num_labels)
    counts = torch.zeros((n_outer * num_labels if samplewise else num_labels, 4), dtype=torch.int64, device=DEV)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    rc = _native.lib().mb200_binary_stat_counts(
        preds.data_ptr(), _native.tag(preds), target.data_ptr(), _native.tag(target), n_outer, num_labels, inner,
        ctypes.c_double(float(threshold)), int(ignore_index is not None), int(ignore_index or 0), int(samplewise),
        counts.data_ptr(), flag.data_ptr(), None, _native.stream_handle(torch.device(DEV)))
    _native.check(rc, "binary_stat_counts")
    return counts


def check(preds, target, num_labels, threshold, ignore_index, samplewise, path, small=True):
    """Kernel == chain, exactly, on the asserted path."""
    assert path_of(preds, target, num_labels, samplewise) == (path, small), (preds.dtype, preds.shape, target.dtype)
    got = kernel(preds, target, num_labels, threshold, ignore_index, samplewise)
    want = ob.stat_counts(preds, target, threshold, ignore_index, num_labels > 1 or preds.ndim == 3, samplewise)
    assert torch.equal(got, want), (path, preds.dtype, threshold, ignore_index, (got - want).abs().sum(0).tolist())
    return got


# ------------------------------------------------------------------------------------------------------------------
# scores
# ------------------------------------------------------------------------------------------------------------------
def every_pattern(dtype) -> torch.Tensor:
    """All 65 536 values of a 16-bit float dtype, NaNs and infinities included."""
    return torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(dtype)


def ulp_window(x: float, dtype, k: int) -> torch.Tensor:
    """x rounded to `dtype` and the k neighbours on each side (finite ones)."""
    itype = torch.int64 if dtype == torch.float64 else torch.int32
    c = torch.tensor([x], dtype=torch.float64).to(dtype)
    # stepping the bit pattern moves away from zero on both signs, so +-k covers both sides; crossing zero gives NaNs
    w = (c.view(itype) + torch.arange(-k, k + 1, dtype=itype)).view(dtype)
    return w[torch.isfinite(w)]


def batch(dtype, threshold: float, kind: str, seed: int = 0) -> torch.Tensor:
    """1-D scores on the device.  `logits` batches hold scores outside [0, 1]; `probs` batches do not."""
    g = torch.Generator().manual_seed(seed + int(threshold * 1e6))
    if dtype in HALF:
        x = every_pattern(dtype)
        if kind == "probs":
            x = x[(x >= 0) & (x <= 1)]
        elif kind == "probs_nan":
            x = x[((x >= 0) & (x <= 1)) | torch.isnan(x)]
        return x[torch.randperm(x.numel(), generator=g)].to(DEV)
    if kind == "probs":
        parts = [ulp_window(threshold, dtype, 64).clamp(0, 1), torch.rand(1 << 16, generator=g, dtype=torch.float64)]
    else:
        if 0.0 < threshold < 1.0:
            c = math.log(threshold / (1 - threshold))
            parts = [ulp_window(c, dtype, 64), c + torch.linspace(-1, 1, 4097, dtype=torch.float64) * 1e-3 * (1 + abs(c))]
        else:
            parts = [torch.tensor([-100.0, -40.0, -17.0, 17.0, 40.0, 100.0], dtype=torch.float64)]
        parts.append(torch.randn(1 << 16, generator=g, dtype=torch.float64) * 6)
    x = torch.cat([p.to(dtype) for p in parts])
    return x[torch.randperm(x.numel(), generator=g)].to(DEV)


def labels(shape, ignore_index=None, dtype=torch.int64, seed: int = 1) -> torch.Tensor:
    """Random {0, 1} targets; with ignore_index -1 an eighth of them are -1."""
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, 2, shape, generator=g)
    if ignore_index == -1:
        t[torch.rand(shape, generator=g) < 0.125] = -1
    return t.to(dtype).to(DEV)


def as_rows(x: torch.Tensor, width: int) -> torch.Tensor:
    """x as [N, width], wrapping around so that every score is kept."""
    n = -(-x.numel() // width)
    return torch.cat([x, x[: n * width - x.numel()]]).reshape(n, width)


# ------------------------------------------------------------------------------------------------------------------
# launch paths
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,threshold", CASES, ids=CASE_IDS)
def test_binary_flat_paths(dtype, threshold):
    """Binary, global, int64 targets, aligned: the single pass (the two-pass flat kernel for float64), bit-identical to
    the two-pass entry and to the chain."""
    for kind in KINDS.get(dtype, ("logits", "probs")):
        x = batch(dtype, threshold, kind)
        assert ob.is_logits(x) == (kind == "logits")
        for ign in (None, -1, 0, 1):
            t = labels(x.shape, ign)
            got = check(x, t, 1, threshold, ign, False, "two_pass" if dtype == torch.float64 else "single_pass")
            if dtype != torch.float64:
                assert path_of(x, t, 1, False, large_scratch=False) == ("two_pass", True)
                assert torch.equal(two_pass(x, t, 1, threshold, ign, False), got), (kind, ign)


@pytest.mark.parametrize("dtype,threshold", CASES, ids=CASE_IDS)
def test_multilabel_column_owner(dtype, threshold):
    for kind in ("logits", "probs"):
        x1 = batch(dtype, threshold, kind, seed=2)
        for L in (2, 3, 37, 128, 129, 255, 256):
            x = as_rows(x1, L)
            for ign in (None, -1):
                check(x, labels(x.shape, ign, seed=L), L, threshold, ign, False, "columns")


@pytest.mark.parametrize("dtype,threshold", CASES, ids=CASE_IDS)
def test_generic_shared_memory_groups(dtype, threshold):
    for kind in ("logits", "probs"):
        x1 = batch(dtype, threshold, kind, seed=3)
        for L in (257, 2048):  # too many labels for the column owner
            x = as_rows(x1, L)
            check(x, labels(x.shape, -1), L, threshold, -1, False, "generic_shared")
        x = as_rows(x1, 3 * 64).reshape(-1, 3, 64)  # inner > 1, global and samplewise (N * 3 <= 2048 groups)
        assert x.shape[0] * 3 <= SMEM_GROUPS
        for ign in (None, 0):
            t = labels(x.shape, ign)
            check(x, t, 3, threshold, ign, False, "generic_shared")
            check(x, t, 3, threshold, ign, True, "generic_shared")
        xb = as_rows(x1, 1024)  # binary samplewise
        check(xb, labels(xb.shape, -1), 1, threshold, -1, True, "generic_shared")
        t = labels(x1.shape, 1, dtype=torch.int32)  # binary global with a non-int64 target
        check(x1, t, 1, threshold, 1, False, "generic_shared")
        buf = torch.cat([x1[:1], x1])  # a view one element past a 16-byte boundary
        xm = buf[1:]
        assert xm.data_ptr() % 16 != 0
        check(xm, labels(xm.shape, -1), 1, threshold, -1, False, "generic_shared")


@pytest.mark.parametrize("dtype,threshold", CASES, ids=CASE_IDS)
def test_generic_global_atomics(dtype, threshold):
    for kind in ("logits", "probs"):
        x1 = batch(dtype, threshold, kind, seed=4)
        xb = as_rows(x1, 4)  # binary samplewise: one group per row
        assert xb.shape[0] > SMEM_GROUPS
        check(xb, labels(xb.shape, -1), 1, threshold, -1, True, "generic_global")
        x = as_rows(x1, 3 * 2).reshape(-1, 3, 2)
        assert x.shape[0] * 3 > SMEM_GROUPS
        check(x, labels(x.shape, 0), 3, threshold, 0, True, "generic_global")
        xl = as_rows(x1, 3000)  # more labels than shared memory holds, global
        check(xl, labels(xl.shape), 3000, threshold, None, False, "generic_global")


@pytest.mark.parametrize("target_dtype", [torch.int64, torch.int32, torch.int16, torch.int8, torch.uint8, torch.bool])
@pytest.mark.parametrize("ign", [None, -1, 0, 1])
def test_target_dtypes(target_dtype, ign):
    if target_dtype == torch.bool and ign in (0, 1):
        pytest.skip("the reference's `target[idx] = -1` stores True into a bool target: it counts ignored elements")
    for dtype, threshold in ((torch.bfloat16, 0.3), (torch.float16, 0.9999), (torch.float32, 1 / 3)):
        for kind in ("logits", "probs"):
            x = batch(dtype, threshold, kind, seed=5)
            t = labels(x.shape, ign if target_dtype.is_signed else None, target_dtype)
            path = "single_pass" if target_dtype == torch.int64 else "generic_shared"
            check(x, t, 1, threshold, ign, False, path)
            xs = as_rows(x, 4)
            ts = labels(xs.shape, ign if target_dtype.is_signed else None, target_dtype)
            check(xs, ts, 1, threshold, ign, True, "generic_global")
            xm = as_rows(x, 37)
            check(xm, labels(xm.shape, ign if target_dtype.is_signed else None, target_dtype), 37, threshold, ign, False,
                  "columns")


def test_float_target_through_the_functional():
    """A float 0. / 1. target is cast to int64 in Python before the kernel (functional/classification/_binary_counts.py)."""
    from metrics_b200.functional.classification import binary_stat_scores

    x = batch(torch.bfloat16, 0.3, "probs", seed=6)
    t = labels(x.shape)
    got = binary_stat_scores(x, t.float(), threshold=0.3)
    want = ob.stat_counts(x, t.float(), 0.3)
    assert torch.equal(got[:4], want[0])


@pytest.mark.parametrize("pred_dtype", [torch.int64, torch.int32, torch.uint8, torch.bool])
def test_integer_label_predictions(pred_dtype):
    g = torch.Generator().manual_seed(7)
    p = torch.randint(0, 2, (4096, 12), generator=g).to(pred_dtype).to(DEV)
    for ign in (None, -1):
        t = labels(p.shape, ign)
        check(p, t, 1, 0.3, ign, False, "labels_shared")
        check(p, t, 1, 0.3, ign, True, "labels_global")
        check(p, t, 12, 0.3, ign, False, "labels_shared")
        check(p.reshape(-1, 3, 4), t.reshape(-1, 3, 4), 3, 0.3, ign, True, "labels_global")
    if pred_dtype == torch.bool:
        return
    bad = p.clone()
    bad[5, 3] = 2  # out of range: flagged, and counted like the reference counts it (a mismatch)
    t = labels(p.shape)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    got = kernel(bad, t, 1, 0.5, None, False, flag)
    assert int(flag.item()) & _native.FLAG_PREDS_RANGE
    assert torch.equal(got, ob.stat_counts(bad, t))
    flag.zero_()
    kernel(p, t, 1, 0.5, None, False, flag)
    assert int(flag.item()) == 0


def test_64bit_index_arithmetic():
    """At least 2^31 elements in `[N, 3, K]` layout: the generic kernel's 64-bit index path (the sample and label of an
    element need 64-bit divisions), on a misaligned bfloat16 view with uint8 targets.  The chain runs in row chunks under
    the vote of the whole batch; global counts of the chunks add up, samplewise ones concatenate."""
    K = 1024
    N = -(-(1 << 31) // (3 * K))
    need = N * 3 * K * 6 + (4 << 30)  # scores (2 B), targets (1 B), the vote's temporaries (3 B), the chain's chunks
    if torch.cuda.mem_get_info(DEV)[0] < need:
        pytest.skip(f"needs {need >> 30} GiB of free device memory")
    g = torch.Generator(device=DEV).manual_seed(8)
    buf = torch.randn(N * 3 * K + 1, generator=g, device=DEV, dtype=torch.bfloat16)
    x = buf[1:].view(N, 3, K)
    t = torch.randint(0, 2, (N, 3, K), generator=g, device=DEV, dtype=torch.uint8)
    assert x.data_ptr() % 16 != 0 and x.numel() >= 2**31
    threshold = 0.3
    vote = ob.is_logits(x)
    assert vote
    for samplewise in (False, True):
        path = "generic_global" if samplewise else "generic_shared"
        assert path_of(x, t, 3, samplewise) == (path, False)
        got = kernel(x, t, 3, threshold, None, samplewise)
        rows = 1 << 16
        parts = [ob.stat_counts(x[r: r + rows], t[r: r + rows], threshold, None, True, samplewise, logits=vote)
                 for r in range(0, N, rows)]
        want = torch.cat(parts) if samplewise else torch.stack(parts).sum(0)
        assert torch.equal(got, want), (samplewise, (got - want).abs().sum(0).tolist())
        del got, parts, want


# ------------------------------------------------------------------------------------------------------------------
# public entry points at a threshold half precision cannot represent
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", HALF)
def test_public_entry_points(dtype):
    import metrics_b200.functional.classification as fc
    from metrics_b200.classification import BinaryStatScores

    thr = 0.3
    x = batch(dtype, thr, "probs", seed=9)
    t = labels(x.shape)
    c = ob.stat_counts(x, t, thr)[0]
    assert torch.equal(fc.binary_stat_scores(x, t, threshold=thr), torch.cat([c, c[:1] + c[3:]]))
    tp, fp, tn, fn = c.tolist()
    assert fc.binary_confusion_matrix(x, t, threshold=thr).tolist() == [[tn, fp], [fn, tp]]
    xs, ts = as_rows(x, 64), as_rows(t, 64)
    sw = ob.stat_counts(xs, ts, thr, samplewise=True)
    got = fc.binary_stat_scores(xs, ts, threshold=thr, multidim_average="samplewise")
    assert torch.equal(got[:, :4], sw)

    xl, tl = as_rows(x, 6), as_rows(t, 6)
    cl = ob.stat_counts(xl, tl, thr, multilabel=True)
    got = fc.multilabel_stat_scores(xl, tl, 6, threshold=thr, average="none")
    assert torch.equal(got[:, :4], cl)
    cm = fc.multilabel_confusion_matrix(xl, tl, 6, threshold=thr)
    assert torch.equal(cm, torch.stack([cl[:, 2], cl[:, 1], cl[:, 3], cl[:, 0]], -1).reshape(6, 2, 2))

    logits = batch(dtype, thr, "logits", seed=10)
    m = BinaryStatScores(threshold=thr).to(DEV)
    want = torch.zeros(4, dtype=torch.int64, device=DEV)
    xx = torch.cat([x, logits])
    for chunk, tc in zip(torch.tensor_split(xx, 5), torch.tensor_split(labels(xx.shape), 5)):
        m.update(chunk, tc)
        want += ob.stat_counts(chunk, tc, thr)[0]  # the logits vote is per update
    assert torch.equal(m.compute()[:4], want)

    groups = torch.randint(0, 3, x.shape, generator=torch.Generator().manual_seed(11)).to(DEV)
    rates = fc.binary_groups_stat_rates(x, t, groups, 3, threshold=thr)
    for gid in range(3):
        sel = groups == gid
        cg = ob.stat_counts(x[sel], t[sel], thr)[0]
        assert torch.equal(rates[f"group_{gid}"], cg / cg.sum()), gid
