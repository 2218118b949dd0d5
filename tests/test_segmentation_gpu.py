"""GPU: kernel K15 (segmentation overlap counts) against the numpy oracle, the reference's goldens through the three classes
and functionals, out-of-range labels, host synchronisation and launch counts, counts above 2^32, and the runtime."""
import numpy as np
import pytest
import torch

from oracle import segmentation as osg
from tests import segmentation_cases as sc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
INT_DTYPES = (torch.bool, torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64)
FLOAT_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def k15(preds, target, num_classes, index, mul, include_background):
    from metrics_b200 import _native

    flag = torch.zeros(1, dtype=torch.int32, device=preds.device) if index else None
    out = _native.segmentation_overlap_counts(preds, target, num_classes, index, mul, not include_background, flag)
    return out.cpu(), None if flag is None else int(flag.item())


def want_counts(preds, target, num_classes, index, mul, include_background):
    """The numpy oracle; bfloat16 (no numpy dtype) through the torch op chain on CPU with float64 sums."""
    p, t = preds.cpu(), target.cpu()
    if p.dtype == torch.bfloat16:
        if not include_background and p.shape[1] > 1:
            p, t = p[:, 1:], t[:, 1:]
        axes = list(range(2, p.ndim))
        return [x.double().sum(dim=axes).numpy() for x in (p * t, p, t)]
    return osg.counts(p.numpy(), t.numpy(), num_classes, include_background, index, "mul" if mul else "and")


def check(preds, target, num_classes, index, mul=True, include_background=True):
    got, flag = k15(preds, target, num_classes, index, mul, include_background)
    want = want_counts(preds, target, num_classes, index, mul, include_background)
    for g, w, name in zip(got, want, ("intersection", "pred_sum", "target_sum")):
        if got.dtype == torch.float64:
            np.testing.assert_allclose(g.numpy(), w, rtol=1e-12, err_msg=name)
        else:
            assert np.array_equal(g.numpy(), w), (name, preds.dtype, tuple(preds.shape), num_classes, include_background)
    return flag


def coherent_labels(g, n, shape, c, block=8):
    small = torch.randint(0, c, (n, *shape[:-1], (shape[-1] + block - 1) // block), generator=g)
    return small.repeat_interleave(block, -1)[..., : shape[-1]].contiguous()


def one_hot_values(g, n, c, shape, dtype, binary=True):
    if binary:
        x = torch.nn.functional.one_hot(torch.randint(0, c, (n, *shape), generator=g), c).movedim(-1, 1).contiguous()
        x = x | (torch.rand(x.shape, generator=g) < 0.1)
    elif dtype.is_floating_point:
        x = torch.randn((n, c, *shape), generator=g) * 3
    else:
        x = torch.randint(-128 if dtype != torch.uint8 else 0, 128 if dtype != torch.uint8 else 256, (n, c, *shape), generator=g)
    return x.to(dtype)


# ---- index format ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [1, 2, 19, 150, 4096, 4097, 9000])
@pytest.mark.parametrize("bg", [True, False])
def test_index_counts_every_class_count(C, bg):
    g = torch.Generator().manual_seed(C * 2 + bg)
    p = coherent_labels(g, 3, (37, 41), C)
    t = torch.where(torch.rand(p.shape, generator=g) < 0.2, torch.randint(0, C, p.shape, generator=g), p)
    assert check(p.to(DEV), t.to(DEV), C, True, include_background=bg) == 0


@pytest.mark.parametrize("inner", [1, 3, 15, 16, 17, 1023, 1024, 1025, 8191, 8193, 100003])
def test_index_counts_at_size_edges_and_offsets(inner):
    g = torch.Generator().manual_seed(inner)
    base = torch.randint(0, 7, (2 * inner + 1,), generator=g).to(DEV)
    tb = torch.randint(0, 7, (2 * inner + 1,), generator=g).to(DEV)
    for off in (0, 1):  # one-element offset views of device memory: 8-byte but not 16-byte aligned
        p, t = base[off:off + 2 * inner].view(2, inner), tb[off:off + 2 * inner].view(2, inner)
        check(p, t, 7, True)
        check(p[:, None], t[:, None], 7, True, include_background=False)


@pytest.mark.parametrize("shape", [(500,), (24, 31), (5, 9, 13)])
def test_index_counts_spatial_ranks_single_class_and_background(shape):
    g = torch.Generator().manual_seed(len(shape))
    p = torch.randint(0, 19, (4, *shape), generator=g)
    check(p.to(DEV), p.flip(0).to(DEV), 19, True)
    one = torch.full((3, *shape), 5)  # every warp holds one class: the worst atomic conflict
    check(one.to(DEV), one.to(DEV), 19, True)
    zero = torch.zeros((3, *shape), dtype=torch.long)  # all background, dropped
    got, _ = k15(zero.to(DEV), zero.to(DEV), 19, True, True, False)
    assert not got.any()
    got, _ = k15(zero.to(DEV), zero.to(DEV), 19, True, True, True)
    assert (got[:, :, 0] == int(np.prod(shape))).all() and not got[:, :, 1:].any()


# ---- one-hot format ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", INT_DTYPES + FLOAT_DTYPES)
@pytest.mark.parametrize("layout", ["planar", "channels_last", "strided"])
def test_one_hot_counts_every_dtype_and_layout(dtype, layout):
    g = torch.Generator().manual_seed(INT_DTYPES.index(dtype) if dtype in INT_DTYPES else 10 + FLOAT_DTYPES.index(dtype))
    for binary in (True, False):
        for c, shape in ((1, (40,)), (4, (9, 11)), (19, (3, 5, 7)), (150, (33,))):
            x, y = one_hot_values(g, 3, c, shape, dtype, binary), one_hot_values(g, 3, c, shape, dtype, binary)
            if layout == "channels_last":
                x, y = (v.movedim(1, -1).contiguous().movedim(-1, 1) for v in (x, y))
            xd, yd = x.to(DEV), y.to(DEV)
            if layout == "strided":  # batch-strided views, read in place
                xd, yd = torch.cat([xd, xd])[::2], torch.cat([yd, yd])[::2]
            for bg in (True, False):
                check(xd, yd, c, False, True, bg)
                if not dtype.is_floating_point:
                    check(xd, yd, c, False, False, bg)


@pytest.mark.parametrize("inner", [1, 3, 15, 16, 17, 1023, 1024, 1025, 16383, 16385, 70001])
@pytest.mark.parametrize("dtype", [torch.bool, torch.int32, torch.float16])
def test_one_hot_counts_at_vector_and_tile_edges_and_offsets(inner, dtype):
    g = torch.Generator().manual_seed(inner)
    c = 3
    flat = one_hot_values(g, 1, 2 * c * inner + 1, (1,), dtype).reshape(-1).to(DEV)
    flat2 = one_hot_values(g, 1, 2 * c * inner + 1, (1,), dtype).reshape(-1).to(DEV)
    for off in (0, 1):  # one-element offset views of device memory
        p = flat[off:off + 2 * c * inner].view(2, c, inner)
        t = flat2[off:off + 2 * c * inner].view(2, c, inner)
        q = flat2[1 - off:1 - off + 2 * c * inner].view(2, c, inner)  # the two inputs aligned differently
        for bg in (True, False):
            check(p, t, c, False, True, bg)
            check(p, q, c, False, True, bg)
        check(p.movedim(1, -1).contiguous().movedim(-1, 1), t.movedim(1, -1).contiguous().movedim(-1, 1), c, False, True, False)


@pytest.mark.parametrize("C", [300, 513])
@pytest.mark.parametrize("dtype", [torch.bool, torch.int32, torch.float16])
def test_channels_last_one_hot_beyond_one_column_pass(C, dtype):
    """More than 256 classes: the channels-last reader walks the columns in passes of 256, the last one partial."""
    g = torch.Generator().manual_seed(C)
    for binary in (True, False):
        x = one_hot_values(g, 2, C, (7, 9), dtype, binary).movedim(1, -1).contiguous().movedim(-1, 1).to(DEV)
        y = one_hot_values(g, 2, C, (7, 9), dtype, binary).movedim(1, -1).contiguous().movedim(-1, 1).to(DEV)
        for bg in (True, False):
            check(x, y, C, False, True, bg)


@pytest.mark.parametrize("layout", ["planar", "channels_last"])
@pytest.mark.parametrize("dtype", FLOAT_DTYPES)
def test_float_planes_split_over_many_ctas(layout, dtype):
    """One large sample (the case one CTA per plane or sample would leave the GPU idle), and a wide class count whose
    channels-last partials hit the cap on parts per sample; both against the oracle, twice for the same bits."""
    g = torch.Generator().manual_seed(17)
    for n, c, shape in ((1, 19, (512, 1024)), (2, 600, (48, 50))):
        x = one_hot_values(g, n, c, shape, dtype, binary=False)
        y = one_hot_values(g, n, c, shape, dtype, binary=False)
        if layout == "channels_last":
            x, y = (v.movedim(1, -1).contiguous().movedim(-1, 1) for v in (x, y))
        xd, yd = x.to(DEV), y.to(DEV)
        for bg in (True, False):
            check(xd, yd, c, False, True, bg)
        assert torch.equal(k15(xd, yd, c, False, True, False)[0], k15(xd, yd, c, False, True, False)[0])


def test_float_sums_are_deterministic():
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 5, 300, 301, generator=g).to(DEV)
    y = torch.randn(2, 5, 300, 301, generator=g).to(DEV)
    a, _ = k15(x, y, 5, False, True, True)
    b, _ = k15(x, y, 5, False, True, True)
    assert torch.equal(a, b)
    cl = (x.movedim(1, -1).contiguous().movedim(-1, 1), y.movedim(1, -1).contiguous().movedim(-1, 1))
    assert torch.equal(k15(*cl, 5, False, True, True)[0], k15(*cl, 5, False, True, True)[0])


# ---- goldens -----------------------------------------------------------------------------------------------------------
def test_goldens_through_classes_and_functionals():
    golden = sc.load()
    for key, case in sc.cases(golden, DEV):
        sc.check_case(golden, key, case, DEV)


def test_goldens_in_bfloat16_dice():
    from metrics_b200.functional.segmentation import dice_score

    g = torch.Generator().manual_seed(3)
    p = one_hot_values(g, 3, 4, (9, 9), torch.bfloat16)
    t = one_hot_values(g, 3, 4, (9, 9), torch.bfloat16)
    got = dice_score(p.to(DEV), t.to(DEV), 4, average="none").cpu()
    want = osg.dice_compute_chain(*osg.dice_update_chain(p, t, 4, True, False), "none")
    assert torch.equal(got, want)


# ---- out-of-range labels -----------------------------------------------------------------------------------------------
def test_out_of_range_labels_raise_the_reference_messages_in_order():
    from metrics_b200.segmentation import DiceScore, GeneralizedDiceScore, MeanIoU

    lab = torch.randint(0, 4, (2, 33, 35)).to(DEV)
    neg, big = lab.clone(), lab.clone()
    neg[0, 1, 1], big[1, 20, 2] = -1, 4
    both = neg.clone()
    both[1, 2, 2] = 7
    neg_msg, big_msg = "Class values must be non-negative.", "Class values must be smaller than num_classes."
    cases = [((neg, lab), neg_msg), ((big, lab), big_msg), ((lab, neg), neg_msg), ((lab, big), big_msg),
             ((both, big), neg_msg), ((big, neg), big_msg), ((lab, both), neg_msg)]
    for cls in (MeanIoU, DiceScore, GeneralizedDiceScore):
        m = cls(4, input_format="index").to(DEV)
        m.update(lab, lab)
        before = {k: (torch.cat(v) if isinstance(v, list) else v).clone() for k, v in m.metric_state.items()}
        for (p, t), msg in cases:
            with pytest.raises(RuntimeError) as info:
                m.update(p, t)
            assert str(info.value) == msg, (cls.__name__, msg)
        after = {k: torch.cat(v) if isinstance(v, list) else v for k, v in m.metric_state.items()}
        assert all(torch.equal(before[k], after[k]) for k in before)
    torch.cuda.synchronize()  # no device fault was left behind
    assert int((lab + 1).sum()) == int(lab.sum()) + lab.numel()


# ---- synchronisation and launches ------------------------------------------------------------------------------------
def test_one_hot_updates_do_not_sync_and_launch_k15_once():
    from metrics_b200 import _native
    from metrics_b200.segmentation import DiceScore, GeneralizedDiceScore, MeanIoU

    g = torch.Generator().manual_seed(9)
    x = one_hot_values(g, 4, 6, (20, 20), torch.bool).to(DEV)
    y = one_hot_values(g, 4, 6, (20, 20), torch.bool).to(DEV)
    xh, yh = x.half(), y.half()
    metrics = [MeanIoU(6), DiceScore(6, average="weighted"), GeneralizedDiceScore(6, weight_type="simple"),
               GeneralizedDiceScore(6, include_background=False, per_class=True)]
    metrics = [m.to(DEV) for m in metrics]
    for m in metrics:
        m.update(x, y)  # warm-up (first-call allocations)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for m in metrics:
            for args in ((x, y), (x.movedim(1, -1).contiguous().movedim(-1, 1), y)):
                n0 = _native.launch_count()
                m.update(*args)
                assert _native.launch_count() - n0 == 1, type(m).__name__
        for m in metrics[1:]:
            n0 = _native.launch_count()
            m.update(xh, yh)
            assert _native.launch_count() - n0 == 1
    finally:
        torch.cuda.set_sync_debug_mode("default")
    lab = torch.randint(0, 6, (4, 20, 20)).to(DEV)
    m = DiceScore(6, input_format="index").to(DEV)
    n0 = _native.launch_count()
    m.update(lab, lab)
    assert _native.launch_count() - n0 == 1


# ---- large inputs ------------------------------------------------------------------------------------------------------
def _free_bytes() -> int:
    return torch.cuda.mem_get_info()[0]


def test_one_hot_count_above_2_pow_32():
    n = 2**32 + 3
    if _free_bytes() < n + (1 << 30):
        pytest.skip("not enough free device memory")
    x = torch.ones((1, 1, n), dtype=torch.bool, device=DEV)
    x[0, 0, ::5] = False
    got, _ = k15(x, x, 1, False, True, True)
    ones = n - (n + 4) // 5
    assert got.reshape(-1).tolist() == [ones] * 3
    del x
    torch.cuda.empty_cache()


def test_index_labels_beyond_2_pow_31():
    n = 2**31 + 5
    if _free_bytes() < 8 * n + (1 << 30):
        pytest.skip("not enough free device memory")
    x = torch.ones((1, n), dtype=torch.long, device=DEV)
    x[0, ::7] = 0
    x[0, n - 1] = 2
    got, flag = k15(x, x, 3, True, True, True)
    zeros = (n + 6) // 7 - (1 if (n - 1) % 7 == 0 else 0)
    want = [zeros, n - zeros - 1, 1]
    assert flag == 0 and all(got[k, 0].tolist() == want for k in range(3))
    del x
    torch.cuda.empty_cache()


# ---- runtime -----------------------------------------------------------------------------------------------------------
def test_collection_forward_state_dict_and_reset():
    from metrics_b200 import MetricCollection
    from metrics_b200.segmentation import DiceScore, GeneralizedDiceScore, MeanIoU

    g = torch.Generator().manual_seed(11)
    batches = [(torch.randint(0, 5, (3, 16, 16), generator=g).to(DEV), torch.randint(0, 5, (3, 16, 16), generator=g).to(DEV))
               for _ in range(3)]
    kw = dict(num_classes=5, input_format="index")
    col = MetricCollection({"miou": MeanIoU(**kw), "dice": DiceScore(**kw), "gdice": GeneralizedDiceScore(**kw)}).to(DEV)
    for p, t in batches:
        step = col(p, t)
        assert set(step) == {"miou", "dice", "gdice"}
    res = col.compute()
    want_miou = np.mean([osg.mean_iou_scores(*osg.counts(p.cpu().numpy(), t.cpu().numpy(), 5, True, True, "and"), False).mean()
                         for p, t in batches])
    assert abs(float(res["miou"]) - want_miou) < 1e-6
    sd = col.state_dict()
    fresh = MetricCollection({"miou": MeanIoU(**kw), "dice": DiceScore(**kw), "gdice": GeneralizedDiceScore(**kw)}).to(DEV)
    for m in (*col.values(), *fresh.values()):
        m.persistent(True)
    fresh.load_state_dict(col.state_dict())
    assert {k: float(v) for k, v in fresh.compute().items()} == pytest.approx({k: float(v) for k, v in res.items()}, rel=1e-6)
    col.reset()
    assert int(col["miou"].num_batches) == 0 and float(col["gdice"].samples) == 0 and sd is not None
