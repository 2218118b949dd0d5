"""GPU: the single-pass binary counting kernel (csrc/binary.cu `bin_count_flat_both_kernel`: both outcomes of the logits vote
counted in one read, sigmoid(x) > thr decided by a host-computed bracket around logit(thr)) is bit-identical to the two-pass
kernels behind `mb200_binary_stat_counts` (vote pass, then counting with the exact float32 sigmoid of ATen) — in particular
for scores crowded around the threshold crossing, where the bracket hands over to the exact arithmetic — and to the
reference's rule: the score in its own dtype compared with the threshold rounded to that dtype, as ATen rounds the scalar."""
import ctypes
import math

import pytest
import torch

from metrics_b200 import _native

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _two_pass(preds, target, threshold, ignore_index):
    """The original entry point (4-byte vote word: two passes over the scores)."""
    counts = torch.zeros((1, 4), dtype=torch.int64, device=DEV)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    rc = _native.lib().mb200_binary_stat_counts(
        preds.data_ptr(), _native.tag(preds), target.data_ptr(), _native.tag(target), preds.numel(), 1, 1,
        ctypes.c_double(float(threshold)), int(ignore_index is not None), int(ignore_index or 0), 0, counts.data_ptr(),
        flag.data_ptr(), None, _native.stream_handle(torch.device(DEV)))
    _native.check(rc, "binary_stat_counts")
    return counts


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("threshold", [0.5, 0.1, 0.9, 0.999, 1e-4, 0.0, 1.0, 0.3333333,
                                       # not representable in half precision: bf16(0.3) = 0.30078125, bf16(0.9999) = 1.0
                                       0.3, 0.7, 0.9999,
                                       # float16 subnormal range: the spacing (2^-24) exceeds thr * 2^-9
                                       2e-6, 1.2e-5, 3e-5, 6e-5,
                                       # rounded to float32 first, these fall on the other side of a half-precision midpoint
                                       0.5 + 2**-12 + 2**-40, 0.5 + 2**-9 + 2**-40])
@pytest.mark.parametrize("kind", ["logits", "probs"])
def test_single_pass_equals_two_pass(dtype, threshold, kind):
    n = 1 << 18
    g = torch.Generator().manual_seed(int(threshold * 1000) + 7)
    if kind == "logits":
        x = torch.randn(n, generator=g) * 4
        if 0.0 < threshold < 1.0:  # crowd the crossing: logit(thr) +- a few ulps of T, and a coarse neighbourhood
            c = math.log(threshold / (1 - threshold))
            near = c + (torch.rand(n // 4, generator=g) - 0.5) * 0.2 * (1 + abs(c))
            x[: n // 4] = near
            x[n // 4: n // 4 + 4096] = torch.tensor(c).to(dtype).float() + torch.arange(-2048, 2048) * torch.finfo(dtype).eps * max(1.0, abs(c))
    else:
        x = torch.rand(n, generator=g)
        x[:4096] = threshold  # exactly on the threshold: `>` is false
    x = x.to(dtype).to(DEV)
    t = torch.randint(0, 2, (n,), generator=g).to(DEV)
    t[100:140] = -1
    for ignore in (None, -1):
        got = _native.binary_stat_counts(x, t, 1, threshold, ignore, False)
        want = _two_pass(x, t, threshold, ignore)
        assert torch.equal(got, want), (got, want)
    # oracle: the reference's rule — the score (for logits its float32 sigmoid stored in T) compared in T with the Python
    # float, which ATen rounds to T first
    xs = torch.sigmoid(x) if kind == "logits" else x  # ATen CUDA sigmoid == K6 (tests/test_normalize_aten_gpu.py)
    p = (xs > threshold).long().cpu()
    tt = t.cpu()
    keep = tt != -1
    exp = [int(((p == 1) & (tt == 1) & keep).sum()), int(((p == 1) & (tt == 0) & keep).sum()),
           int(((p == 0) & (tt == 0) & keep).sum()), int(((p == 0) & (tt == 1) & keep).sum())]
    assert _native.binary_stat_counts(x, t, 1, threshold, -1, False).cpu().reshape(-1).tolist() == exp


def test_nan_and_infinite_scores():
    x = torch.tensor([float("nan"), float("inf"), float("-inf"), 0.3, -0.0, 2.0] * 1000, device=DEV)
    t = torch.tensor([1, 1, 0, 0, 1, 0] * 1000, device=DEV)
    assert torch.equal(_native.binary_stat_counts(x, t, 1, 0.5, None, False), _two_pass(x, t, 0.5, None))
