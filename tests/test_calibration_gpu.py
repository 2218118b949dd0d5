"""GPU: calibration error — kernel K14a against the reference's op chain on the same GPU (oracle/calibration.py), kernel
K14b and the epilogue against the reference's goldens and the float64 oracle, and the metric classes' plumbing."""
import os

import numpy as np
import pytest
import torch

from oracle import calibration as oc
from tests.conftest import GOLDEN_DIR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = {0: torch.float32, 1: torch.float16, 2: torch.bfloat16, 3: torch.float64}


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.float().contiguous().view(torch.int32)


def crafted_rows(C: int, dtype: torch.dtype, g: torch.Generator) -> torch.Tensor:
    """Logit rows whose softmax ties after rounding to `dtype` (the first index must win over the larger logit), NaN rows,
    +-inf, all-equal rows, and the maximum in the first / last column."""
    rows = torch.randn(16, C, generator=g) * 2
    tiny = {torch.float32: 1.4e-45, torch.float16: 6e-8, torch.bfloat16: 1e-38}[dtype]
    rows[0, :] = -3.0
    rows[0, 1], rows[0, C - 1] = 0.0, tiny  # different logits, same rounded probability
    rows[1, :] = -3.0
    rows[1, 0], rows[1, 2 % C] = 1.0, 1.0 + tiny
    rows[2, C // 2] = float("nan")
    rows[3, :] = float("nan")
    rows[4, :] = 0.25
    rows[5, C - 1] = 40.0
    rows[6, 0] = 40.0
    rows[7, 1] = float("inf")
    rows[8, :] = -float("inf")
    rows[9, :] = 7.0
    return rows.to(dtype)


def check_bits(preds, target, num_classes, ignore_index=None):
    from metrics_b200.functional.classification.calibration_error import _multiclass_calibration_error_fused_update

    got_c, got_a = _multiclass_calibration_error_fused_update(preds, target, num_classes, ignore_index)
    want_c, want_a = oc.multiclass_calibration_update_chain(preds, target, num_classes, ignore_index)
    assert got_c.dtype == torch.float32 and got_a.dtype == torch.float32
    assert torch.equal(bits(got_c), bits(want_c)), (preds.dtype, preds.shape, ignore_index)
    assert torch.equal(got_a, want_a), (preds.dtype, preds.shape, ignore_index)


@pytest.mark.parametrize("C", [3, 10, 1000, 1024])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_top_label_is_bit_equal_to_the_aten_chain(C, dtype):
    g = torch.Generator().manual_seed(C * 7 + {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}[dtype])
    n = 3000 if C < 1000 else 600
    logits = torch.cat([torch.randn(n, C, generator=g) * 4, crafted_rows(C, torch.float32, g)]).to(dtype)
    target = torch.randint(0, C, (logits.shape[0],), generator=g)
    target[:16] = torch.arange(16) % C  # crafted rows: hits and misses on the tie positions
    lg, tg = logits.to(DEV), target.to(DEV)
    check_bits(lg, tg, C)
    check_bits(lg, tg, C, ignore_index=-1)
    probs = torch.softmax(lg.float(), 1).to(dtype)
    probs[5, :] = float("nan")  # NaN does not vote: the batch stays probabilities
    probs[6, 0] = probs[6, C - 1] = probs[6].max()  # a tie in the raw probabilities
    check_bits(probs, tg, C)
    # ignored rows hold the only out-of-range scores: without them the batch is probabilities
    flip = probs.clone()
    flip[::7] = lg[::7]
    ig = tg.clone()
    ig[::7] = C + 3
    check_bits(flip, ig, C, ignore_index=C + 3)
    check_bits(flip, tg, C)  # ... and with them it is logits
    # a batch of logits whose rows mostly lie inside [0, 1]: in-range rows take their softmax candidate
    mostly = probs.clone()
    mostly[n // 2] = lg[n // 2] * 10
    check_bits(mostly, tg, C)
    # multidim [N, C, d]
    md = lg[: 40 * 3].reshape(40, 3, C).transpose(1, 2).contiguous()
    check_bits(md, tg[: 120].reshape(40, 3), C)


@pytest.mark.parametrize("C,dtype", [(1025, torch.float32), (4096, torch.bfloat16), (4096, torch.float16),
                                     (10, torch.float64), (1000, torch.float64), (3000, torch.float64)])
def test_top_label_wide_rows_and_float64(C, dtype):
    from metrics_b200.functional.classification.calibration_error import _multiclass_calibration_error_fused_update

    g = torch.Generator().manual_seed(C)
    n = 700
    logits = (torch.randn(n, C, generator=g, dtype=torch.float64) * 4).to(dtype).to(DEV)
    target = torch.randint(0, C, (n,), generator=g).to(DEV)
    target[::9] = -1
    for preds in (logits, torch.softmax(logits.double(), 1).to(dtype)):
        for ignore in (None, -1):
            got_c, got_a = _multiclass_calibration_error_fused_update(preds, target, C, ignore)
            want_c, want_a = oc.multiclass_calibration_update_chain(preds, target, C, ignore)
            torch.testing.assert_close(got_c, want_c, rtol=1e-6, atol=0)
            assert (got_a != want_a).float().mean().item() <= 2e-3


def _golden():
    return np.load(os.path.join(GOLDEN_DIR, "calibration.npz"), allow_pickle=False)


TOL = {torch.float32: 2e-5, torch.float16: 2e-2, torch.bfloat16: 1.5e-1, torch.float64: 1e-12}


def test_classes_against_the_goldens_and_the_float64_oracle():
    from metrics_b200.classification import BinaryCalibrationError, MulticlassCalibrationError

    golden = _golden()
    for k in range(int(golden["n_cases"])):
        key = f"case{k}"
        binary, n_batches, n_bins, ignore, num_classes, code = (int(v) for v in golden[f"{key}/meta"])
        ignore = None if ignore == -999 else ignore
        dtype = DTYPES[code]
        for norm in ("l1", "l2", "max"):
            m = (BinaryCalibrationError(n_bins=n_bins, norm=norm, ignore_index=ignore) if binary
                 else MulticlassCalibrationError(num_classes, n_bins=n_bins, norm=norm, ignore_index=ignore)).to(DEV)
            for b in range(n_batches):
                m.update(torch.from_numpy(golden[f"{key}/preds{b}"]).to(dtype).to(DEV),
                         torch.from_numpy(golden[f"{key}/target{b}"]).to(DEV))
            conf, acc = torch.cat(m.confidences), torch.cat(m.accuracies)
            # the states: same as the reference's up to the last bit of the softmax / sigmoid (CPU vs GPU transcendental)
            np.testing.assert_allclose(conf.float().cpu().numpy(), golden[f"{key}/conf"], rtol=8e-3 if binary else 1e-6,
                                       atol=1e-7, equal_nan=True, err_msg=key)
            assert np.array_equal(acc.float().cpu().numpy(), golden[f"{key}/acc"].astype(np.float32)), key
            got = float(m.compute())
            state_dtype = dtype if binary else torch.float32
            b = torch.linspace(0, 1, n_bins + 1, dtype=conf.dtype).double().numpy()
            want = oc.ce_compute(conf.double().cpu().numpy(), acc.double().cpu().numpy(), b, norm)
            exact = {torch.float32: 2e-6, torch.float16: 2e-3, torch.bfloat16: 1.6e-2, torch.float64: 1e-12}[state_dtype]
            assert abs(got - want) <= exact * max(1.0, abs(want)), (key, norm, got, want)
            assert abs(got - float(golden[f"{key}/{norm}"])) <= 2 * TOL[state_dtype] + 1e-4, (key, norm)


def test_docstring_values_and_l2_zero():
    import metrics_b200.functional.classification as F

    p = torch.tensor([0.25, 0.25, 0.55, 0.75, 0.75], device=DEV)
    t = torch.tensor([0, 0, 1, 1, 1], device=DEV)
    got = [float(F.binary_calibration_error(p, t, n_bins=2, norm=n)) for n in ("l1", "l2", "max")]
    np.testing.assert_allclose(got, _golden()["doc/binary"], rtol=1e-6)
    p = torch.tensor([[0.25, 0.20, 0.55], [0.55, 0.05, 0.40], [0.10, 0.30, 0.60], [0.90, 0.05, 0.05]], device=DEV)
    t = torch.tensor([0, 1, 2, 0], device=DEV)
    got = [float(F.calibration_error(p, t, "multiclass", n_bins=3, norm=n, num_classes=3)) for n in ("l1", "l2", "max")]
    np.testing.assert_allclose(got, _golden()["doc/multiclass"], rtol=1e-6)
    zero = F.binary_calibration_error(torch.tensor([0.0, 0.0, 1.0, 1.0], device=DEV), torch.tensor([0, 0, 1, 1], device=DEV),
                                      n_bins=4, norm="l2")
    assert zero.dtype == torch.int64 and int(zero) == 0 and zero.device.type == "cpu"


def test_bins_beyond_float32_counting():
    """2**24 + 2**22 samples in one bin: the reference's float32 count stops at 2**24; the exact count does not."""
    from metrics_b200.classification import BinaryCalibrationError

    n = (1 << 24) + (1 << 22)
    preds = torch.full((n,), 0.3, device=DEV)
    target = (torch.arange(n, device=DEV) % 3 == 0).long()
    m = BinaryCalibrationError(n_bins=15, validate_args=False).to(DEV)
    m.update(preds, target)
    got = float(m.compute())
    hits = (n + 2) // 3
    want = abs(hits / n - float(torch.tensor(0.3)))
    assert abs(got - want) <= 1e-6, (got, want)
    chain = float(oc.ce_compute_chain(preds, target, 15))
    assert abs(chain - want) > 1e-2, "the reference's float32 bins were expected to lose this count"


def test_binning_is_deterministic_and_matches_the_oracle():
    from metrics_b200 import _native

    g = torch.Generator().manual_seed(99)
    n = 3_000_017
    for dtype, nb in ((torch.float32, 15), (torch.float16, 100), (torch.bfloat16, 7), (torch.float64, 1), (torch.float32, 4000)):
        conf = torch.rand(n, generator=g, dtype=torch.float64).to(dtype)
        conf[::1001] = 1.0
        conf[::997] = float("nan")
        acc = torch.randint(0, 2, (n,), generator=g, dtype=torch.uint8)
        bounds = torch.linspace(0, 1, nb + 1, dtype=dtype)
        conf[5::1003] = bounds[torch.arange(conf[5::1003].numel()) % (nb + 1)]  # exactly on the boundaries
        d_conf, d_acc, d_bounds = conf.to(DEV), acc.to(DEV), bounds.to(DEV)
        first = _native.calibration_bin_sums(d_conf, d_acc, d_bounds)
        second = _native.calibration_bin_sums(d_conf, d_acc, d_bounds)
        for a, b in zip(first, second):
            assert torch.equal(a.view(torch.int64), b.view(torch.int64))
        count, sum_conf, sum_acc = oc.bin_sums(conf.double().numpy(), acc.numpy(), bounds.double().numpy())
        assert np.array_equal(first[0].cpu().numpy(), count), dtype
        np.testing.assert_allclose(first[1].cpu().numpy(), sum_conf, rtol=1e-12, equal_nan=True)
        np.testing.assert_allclose(first[2].cpu().numpy(), sum_acc, rtol=0)


def test_two_computes_give_the_same_bits():
    from metrics_b200.classification import MulticlassCalibrationError

    g = torch.Generator().manual_seed(5)
    m = MulticlassCalibrationError(100, n_bins=15, norm="l2").to(DEV)
    for _ in range(3):
        m.update(torch.randn(20000, 100, generator=g).to(DEV), torch.randint(0, 100, (20000,), generator=g).to(DEV))
    a, b = m.compute(), m.compute()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_update_without_validation_does_not_synchronise():
    from metrics_b200.classification import BinaryCalibrationError, MulticlassCalibrationError

    mc = MulticlassCalibrationError(1000, validate_args=False).to(DEV)
    bc = BinaryCalibrationError(validate_args=False).to(DEV)
    logits = torch.randn(4096, 1000, device=DEV, dtype=torch.bfloat16)
    target = torch.randint(0, 1000, (4096,), device=DEV)
    wide = torch.randn(64, 2000, device=DEV)
    scores = torch.randn(100_000, device=DEV)
    labels = torch.randint(0, 2, (100_000,), device=DEV)
    mc.update(logits, target)  # warm-up (library load, allocator)
    bc.update(scores, labels)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        mc.update(logits, target)
        mc.update(wide.softmax(1)[:, :1000].contiguous(), target[:64])
        bc.update(scores, labels)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert sum(c.numel() for c in mc.confidences) == 2 * 4096 + 64


def test_validation_errors():
    from metrics_b200.classification import BinaryCalibrationError, MulticlassCalibrationError

    m = MulticlassCalibrationError(5).to(DEV)
    with pytest.raises(RuntimeError, match="Detected more unique values in `target`"):
        m.update(torch.randn(10, 5, device=DEV), torch.tensor([0, 1, 2, 3, 4, 5, 0, 1, 2, 3], device=DEV))
    assert m.confidences == []
    m = MulticlassCalibrationError(5, ignore_index=7).to(DEV)
    m.update(torch.randn(10, 5, device=DEV), torch.tensor([0, 1, 2, 3, 4, 7, 0, 1, 2, 3], device=DEV))
    assert m.confidences[0].numel() == 9
    with pytest.raises(ValueError, match="`preds` should be a float tensor"):
        MulticlassCalibrationError(5).update(torch.randint(0, 5, (4, 5), device=DEV), torch.zeros(4, dtype=torch.long, device=DEV))
    with pytest.raises(ValueError, match="Expected argument `preds` to be floating tensor"):
        BinaryCalibrationError().update(torch.randint(0, 2, (4,), device=DEV), torch.zeros(4, dtype=torch.long, device=DEV))
    with pytest.raises(RuntimeError, match="Detected the following values in `target`"):
        BinaryCalibrationError().update(torch.rand(4, device=DEV), torch.tensor([0, 1, 2, 1], device=DEV))
    with pytest.raises(ValueError, match="Expected argument `n_bins` to be an integer larger than 0"):
        BinaryCalibrationError(n_bins=0)
    with pytest.raises(ValueError, match="Expected argument `norm` to be one of"):
        MulticlassCalibrationError(3, norm="l3")


def test_state_dict_collection_and_task_dispatch():
    from metrics_b200 import MetricCollection
    from metrics_b200.classification import (
        BinaryCalibrationError,
        CalibrationError,
        MulticlassAccuracy,
        MulticlassCalibrationError,
    )

    assert isinstance(CalibrationError(task="binary"), BinaryCalibrationError)
    mc = CalibrationError(task="multiclass", num_classes=7, n_bins=10, norm="max")
    assert isinstance(mc, MulticlassCalibrationError) and mc.n_bins == 10 and mc.norm == "max"
    with pytest.raises(ValueError, match="`num_classes` is expected to be `int`"):
        CalibrationError(task="multiclass")

    g = torch.Generator().manual_seed(3)
    preds = torch.randn(500, 7, generator=g).to(DEV)
    target = torch.randint(0, 7, (500,), generator=g).to(DEV)
    mc = mc.to(DEV)
    mc.update(preds, target)
    assert mc.state_dict() == {}  # non-persistent states, like the reference
    mc.persistent(True)
    fresh = MulticlassCalibrationError(7, n_bins=10, norm="max").to(DEV)
    fresh.persistent(True)
    fresh.load_state_dict(mc.state_dict())
    assert torch.equal(fresh.compute(), mc.compute())

    col = MetricCollection([MulticlassCalibrationError(7), MulticlassAccuracy(7)]).to(DEV)
    col.update(preds, target)
    res = col.compute()
    alone = MulticlassCalibrationError(7).to(DEV)
    alone.update(preds, target)
    assert torch.equal(res["MulticlassCalibrationError"], alone.compute())
    assert "MulticlassAccuracy" in res
