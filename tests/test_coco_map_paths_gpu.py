"""GPU: the COCO mAP kernels (K8, csrc/cocomap.cu) and the mask kernels (K12, csrc/maskiou.cu), called through the C-ABI
entries directly, against the record-level restatement of COCOeval (oracle/coco_map.py `match_records`,
`accumulate_records`) and plain numpy bit counting, on every launch path:
  match       register "matched" mask (<= 256 ground truths per image; full at bit 255) and shared-memory mask (257, 700,
              300 over 40 classes); 1, 255, 256, 257 detections and the largest count the 200 KB staging limit admits, one
              past it rejected before launch; (class x area x threshold) work items below and far above 256; T = 1, 10, 16
              (bit 63 of the words); box and mask IoU, micro
  accumulate  per-class record counts around the 256-record tiles and one class of 2^24 + 3 records; K around the radix key
              widths (4 to 7 key bytes); every [class_lo, class_hi) split; permuted records; M = 1..8; recall levels on
              k / npig; nd == 0 with npig > 0 and npig == 0 with detections
  K12         pack: rows around the 2048-pixel warp step, aligned and unaligned, byte values other than 1, the grid cap,
              an output stride wider than a row, hw = 0, more than 2^32 bytes in one call; pairs: D, G = 1..9, empty sides,
              several CTAs per image and the per-image cap, per-image word counts, micro, label mismatch
Every case first asserts the launch path from the launcher's arithmetic, restated here.  Records, `npig`, precision, recall
and scores must be bit-equal (NaN equal to NaN): both sides do the same integer and fp64 operations in the same order.
The NaN-score cases (COCOeval puts NaN last) are the tests named `*nan*`."""

import numpy as np
import pytest
import torch

from metrics_b200 import _native
from oracle.coco_map import accumulate_records, default_rec_thresholds
from tests import coco_map_cases as cases

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SMEM_LIMIT = 200 * 1024
THR16 = torch.linspace(0.5, 0.95, 16).tolist()


# ---- launch arithmetic, restated from the launchers ------------------------------------------------------------------------
def eval_smem_bytes(max_d, max_g):
    """map_match_impl: map_eval_smem_bytes (68 bytes per detection, 52 per ground truth, 64) + the shared "matched" masks."""
    b = 68 * max_d + 52 * max_g + 64
    if max_g > 256:
        b += 256 * ((max_g + 63) // 64) * 8 + 8
    return b


def key_bytes(K):
    """map_accumulate_impl: 4 score bytes + ceil(log256 K) class bytes."""
    b = 0
    while 256 ** b < K:
        b += 1
    return 4 + b


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def t(x, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).to(DEV)


# ---- the match phase ---------------------------------------------------------------------------------------------------------
def run_match(case):
    classes = cases.classes_of(case)
    kw, gt_area = {}, case["gt_area"]
    if "det_masks" in case:
        m = cases.mask_inputs(case)
        gt_area = m["gt_area"]
        kw = dict(gt_area_exact=True, masks={
            "pair_inter": t(np.concatenate([m["pair_inter"], [0.0]]), torch.float64), "pair_off": t(m["pair_off"], torch.int64),
            "det_area": t(m["det_mask_area"], torch.float64), "gt_area": t(m["gt_mask_area"], torch.float64)})
    (cat, rank, match, ignore), npig, err = _native.coco_map_match(
        t(case["det_box"]), t(case["det_score"]), t(case["det_label"]), case["det_counts"], t(case["gt_box"]),
        t(case["gt_label"]), t(case["gt_crowd"]), t(gt_area), case["gt_counts"], t(classes), case["iou_thr"],
        case["max_dets"][-1], micro=case["micro"], **kw)
    return (cat.cpu().numpy(), rank.cpu().numpy(), match.cpu().numpy().view(np.uint64), ignore.cpu().numpy().view(np.uint64),
            npig.cpu().numpy(), int(err.item()))


def check_records(got, want):
    for name, g, w in zip(("det_cat", "det_rank", "det_match", "det_ignore", "npig"), got, want):
        assert g.dtype == w.dtype, name
        np.testing.assert_array_equal(g, w, err_msg=name)
    assert got[5] == 0, "error word"


def run_accumulate(records, score, K, lo, hi, T, rec_thr, max_dets):
    cat, rank, match, ignore, npig = records
    p, r, s, err = _native.coco_map_accumulate(
        t(cat, torch.int32), t(score, torch.float32), t(rank, torch.int32), t(match.view(np.int64), torch.int64),
        t(ignore.view(np.int64), torch.int64), t(npig, torch.int32), K, lo, hi, T, rec_thr, max_dets)
    assert int(err.item()) == 0
    return p.cpu().numpy(), r.cpu().numpy(), s.cpu().numpy()


def check_curves(got, want):
    for name, g, w in zip(("precision", "recall", "scores"), got, want):
        np.testing.assert_array_equal(g, w, err_msg=name)


def check_case(case):
    """match (records) -> accumulate on the kernel's records -> the fused entry (boxes): all bit-equal to the oracle."""
    want = cases.oracle_records(case)
    got = run_match(case)
    check_records(got, want)
    K, T = want[4].shape[0], len(case["iou_thr"])
    want_curves = accumulate_records(*want[:1], case["det_score"], *want[1:], K, 0, K, T, case["rec_thr"], case["max_dets"])
    check_curves(run_accumulate(got[:5], case["det_score"], K, 0, K, T, case["rec_thr"], case["max_dets"]), want_curves)
    if "det_masks" not in case:
        p, r, s, err = _native.coco_map_evaluate(
            t(case["det_box"]), t(case["det_score"]), t(case["det_label"]), case["det_counts"], t(case["gt_box"]),
            t(case["gt_label"]), t(case["gt_crowd"]), t(case["gt_area"]), case["gt_counts"], t(cases.classes_of(case)),
            case["micro"], case["iou_thr"], case["rec_thr"], case["max_dets"])
        assert int(err.item()) == 0
        check_curves((p.cpu().numpy(), r.cpu().numpy(), s.cpu().numpy()), want_curves)
    return got


@pytest.mark.parametrize("name", [n for n in cases.HAND_BUILT if n != "nan_scores"])
def test_hand_built_case(name):
    case = cases.HAND_BUILT[name]()
    assert max(case["gt_counts"]) <= 256 and eval_smem_bytes(max(case["det_counts"]), max(case["gt_counts"])) <= SMEM_LIMIT
    check_case(case)


def test_iou_exactly_at_threshold_matches():
    """float32(0.55) widened is a threshold; IoU == it matches at 0.55, one ulp below does not; 0.5 / 0.75 likewise."""
    case = cases.iou_at_threshold()
    assert case["iou_thr"][1] == cases.F055 / 2 ** 24
    _, _, match, _, _, _ = check_case(case)
    bits = [[int(m) >> b & 1 for b in range(10)] for m in match]  # area "all": bits 0..9
    assert bits[0][:3] == [1, 1, 0] and bits[1][:3] == [1, 0, 0]
    assert bits[2][:2] == [1, 0] and bits[3][5:7] == [1, 0] and bits[4][5:7] == [1, 0]


def test_nan_scores():
    """NaN scores rank after every other score (-inf included) in input order, as COCOeval's mergesort orders them."""
    got = check_case(cases.nan_scores())
    np.testing.assert_array_equal(got[1][:4], [2, 3, 0, 1])


# ---- geometry: random cases at the kernel's path edges --------------------------------------------------------------------
def random_case(seed, det_counts, gt_counts, n_cls, iou_thr, max_dets=(1, 10, 100), crowd=0.1):
    rng = np.random.default_rng(seed)
    sizes = np.array([8, 16, 31, 32, 33, 95, 96, 97, 120], np.float32)
    images = []
    for nd, ng in zip(det_counts, gt_counts):
        gt = []
        for _ in range(ng):
            w, h = rng.choice(sizes, 2)
            area = float(rng.choice([0.0, 0.0, 1024.0, 9216.0, 500.0, 5000.0, 20000.0]))
            gt.append((float(rng.integers(0, 300)), float(rng.integers(0, 300)), float(w), float(h), int(rng.integers(n_cls)),
                       int(rng.random() < crowd), area))
        det = []
        for i in range(nd):
            score = float(rng.integers(0, 24)) / 16
            if gt and rng.random() < 0.6:
                g = gt[int(rng.integers(len(gt)))]
                dx, dy = rng.integers(-4, 5, 2)
                det.append((g[0] + float(dx), g[1] + float(dy), g[2], g[3], score, g[4]))
            else:
                w, h = rng.choice(sizes, 2)
                det.append((float(rng.integers(0, 300)), float(rng.integers(0, 300)), float(w), float(h), score,
                            int(rng.integers(n_cls))))
        images.append(dict(det=det, gt=gt))
    return cases.make_case(images, iou_thr=iou_thr, max_dets=max_dets)


D_MAX = (SMEM_LIMIT - 64 - 52 * 4) // 68  # the most detections per image next to 4 ground truths: 3008

GEOMETRY = {
    # name: (det_counts, gt_counts, classes, thresholds, max_dets, shared-memory mask)
    "gt64": ([20, 5], [64, 3], 1, None, (1, 10, 100), False),
    "gt65": ([20], [65], 1, [0.5], (1, 10, 100), False),
    "gt256_one_class": ([30, 4], [256, 2], 1, [0.5], (1, 10, 100), False),
    "gt257": ([30], [257], 1, [0.5], (1, 10, 100), True),
    "gt700_one_class": ([40, 3], [700, 5], 1, [0.5], (1, 10, 100), True),
    "gt300_40_classes": ([60], [300], 40, None, (1, 10, 100), True),
    "det1": ([1, 0, 1], [3, 2, 0], 2, None, (1, 10, 100), False),
    "det255": ([255, 7], [10, 4], 3, None, (1, 10, 300), False),
    "det256": ([256, 7], [10, 4], 3, None, (1, 10, 300), False),
    "det257": ([257, 7], [10, 4], 3, None, (1, 100, 300), False),
    "det_max": ([D_MAX, 3], [4, 2], 1, [0.5], (1, 10, D_MAX), False),
    "t16": ([50, 40], [30, 20], 4, THR16, (1, 10, 100), False),
    "t1": ([50, 40], [30, 20], 4, [0.5], (1, 10, 100), False),
}


@pytest.mark.parametrize("name", list(GEOMETRY))
def test_match_geometry(name):
    det_counts, gt_counts, n_cls, thr, max_dets, smem_mask = GEOMETRY[name]
    assert (max(gt_counts) > 256) == smem_mask
    assert eval_smem_bytes(max(det_counts), max(gt_counts)) <= SMEM_LIMIT
    check_case(random_case(len(name), det_counts, gt_counts, n_cls, thr, max_dets))


def test_work_items_far_above_block():
    """80 classes x 4 areas x T = 16 = 5120 (class, area, threshold) work items in one image: 20 strided rounds."""
    rng = np.random.default_rng(1)
    det, gt = [], []
    for c in range(80):
        for _ in range(2):
            x, y = (float(v) for v in rng.integers(0, 200, 2))
            gt.append((x, y, 40.0, 40.0, c, 0, 0.0))
            det.append((x + float(rng.integers(0, 8)), y, 40.0, 40.0, float(rng.integers(1, 9)) / 8, c))
    case = cases.make_case([dict(det=det, gt=gt)], iou_thr=THR16)
    assert 80 * 4 * 16 > 256
    check_case(case)


def test_staging_limit_rejected_before_launch():
    case = random_case(2, [D_MAX + 1], [4], 1, [0.5])
    assert eval_smem_bytes(D_MAX + 1, 4) > SMEM_LIMIT >= eval_smem_bytes(D_MAX, 4)
    with pytest.raises(NotImplementedError, match="more than the evaluate kernel can stage"):
        run_match(case)


# ---- the accumulate phase on synthetic records ---------------------------------------------------------------------------
def synth_records(rng, counts, K, T, max_det, npig_max=6):
    """Records of `counts[k]` detections of class k (k < K) in image-like interleaved order, ranks in [0, max_det + 2),
    random match / ignore bits for the 4 * T bits, scores with many ties."""
    cat = np.repeat(np.arange(len(counts), dtype=np.int32), counts)
    rng.shuffle(cat)
    n = len(cat)
    rank = rng.integers(0, max_det + 2, n).astype(np.int32)
    nbits = 4 * T
    mask = np.uint64((1 << nbits) - 1) if nbits < 64 else np.uint64(0xFFFFFFFFFFFFFFFF)
    match = rng.integers(0, 2 ** 63, n, dtype=np.int64).view(np.uint64) << np.uint64(1) | rng.integers(0, 2, n).astype(np.uint64)
    ignore = rng.integers(0, 2 ** 63, n, dtype=np.int64).view(np.uint64) & rng.integers(0, 2 ** 63, n, dtype=np.int64).view(np.uint64)
    score = (rng.integers(0, 64, n) / 64).astype(np.float32)
    npig = rng.integers(0, npig_max, (K, 4)).astype(np.int32)
    return (cat, rank, match & mask, ignore & mask, npig), score


def check_accumulate(records, score, K, T, rec_thr, max_dets, lo=0, hi=None):
    hi = K if hi is None else hi
    want = accumulate_records(records[0], score, *records[1:], K, lo, hi, T, rec_thr, max_dets)
    got = run_accumulate(records, score, K, lo, hi, T, rec_thr, max_dets)
    check_curves(got, want)
    return got


def test_accumulate_tile_edges():
    counts = [1, 255, 256, 257, 511, 512, 513]
    rng = np.random.default_rng(4)
    records, score = synth_records(rng, counts, len(counts), 2, 600)
    records[4][:, :] = np.maximum(records[4], 1)
    check_accumulate(records, score, len(counts), 2, default_rec_thresholds(), [1, 100, 600])


def test_accumulate_one_class_of_2_24_plus_3_records():
    """No float32 may hide in a count: 2^24 + 3 records of one class, T = R = M = 1, ranks around maxDet."""
    n = 2 ** 24 + 3
    rng = np.random.default_rng(6)
    rank = rng.integers(0, n + 2, n).astype(np.int32)
    rank[:5] = n  # exactly maxDet: dropped
    match = rng.integers(0, 2, n).astype(np.uint64)
    ignore = (rng.random(n) < 0.05).astype(np.uint64)
    score = (rng.integers(0, 4096, n) / 4096).astype(np.float32)
    npig = np.array([[2 ** 23 + 5, 0, 0, 0]], np.int32)
    records = (np.zeros(n, np.int32), rank, match, ignore, npig)
    got = check_accumulate(records, score, 1, 1, [0.3712], [n])
    assert got[1][0, 0, 0, 0] > 0


def test_accumulate_empty_sides():
    """nd == 0 with npig > 0 (recall 0, precision / scores 0) and npig == 0 with detections (-1)."""
    rng = np.random.default_rng(8)
    records, score = synth_records(rng, [0, 40, 0], 3, 1, 100)
    records[4][:] = [[3, 0, 1, 0], [0, 0, 0, 0], [1, 1, 1, 1]]
    got = check_accumulate(records, score, 3, 1, [0.0, 0.5, 1.0], [1, 10, 100])
    assert (got[1][0, 0, 0] == 0).all() and (got[1][0, 1] == -1).all()


@pytest.mark.parametrize("K", [1, 2, 256, 257, 65536, 65537])
def test_accumulate_key_width(K):
    """The sort key holds 4 score bytes and ceil(log256 K) class bytes: classes 0, 1, 255, 256, K/2, K - 2, K - 1."""
    assert key_bytes(K) == {1: 4, 2: 5, 256: 5, 257: 6, 65536: 6, 65537: 7}[K]
    rng = np.random.default_rng(K)
    used = sorted({c for c in (0, 1, 255, 256, K // 2, K - 2, K - 1) if 0 <= c < K})
    counts = np.zeros(K, np.int64)
    counts[used] = rng.integers(50, 300, len(used))
    records, score = synth_records(rng, counts, K, 1, 100)
    records[4][:] = 0
    records[4][used] = rng.integers(1, 6, (len(used), 4))
    check_accumulate(records, score, K, 1, [0.5], [100])


def test_accumulate_every_class_range():
    """Sharded accumulation on one GPU: every [lo, hi) equals the full call inside the range and is -1 outside."""
    K, T = 6, 2
    rng = np.random.default_rng(9)
    records, score = synth_records(rng, [30, 0, 300, 5, 260, 1], K, T, 100)
    rec = default_rec_thresholds()
    full = check_accumulate(records, score, K, T, rec, [1, 10, 100])
    for lo in range(K + 1):
        for hi in range(lo, K + 1):
            got = run_accumulate(records, score, K, lo, hi, T, rec, [1, 10, 100])
            for g, f, axis in zip(got, full, (2, 1, 2)):
                want = np.full_like(f, -1.0)
                sl = [slice(None)] * f.ndim
                sl[axis] = slice(lo, hi)
                want[tuple(sl)] = f[tuple(sl)]
                np.testing.assert_array_equal(g, want, err_msg=f"[{lo}, {hi})")


def test_accumulate_permuted_records():
    """Ties in score keep the order the records are given in."""
    rng = np.random.default_rng(10)
    records, score = synth_records(rng, [700, 300], 2, 3, 50)
    perm = rng.permutation(len(score))
    records = tuple(x[perm] for x in records[:4]) + (records[4],)
    check_accumulate(records, score[perm], 2, 3, default_rec_thresholds(), [1, 10, 50])


@pytest.mark.parametrize("M", range(1, 9))
def test_accumulate_max_dets(M):
    rng = np.random.default_rng(20 + M)
    records, score = synth_records(rng, [400, 90], 2, 1, 300)
    check_accumulate(records, score, 2, 1, [0.5], [1, 3, 10, 30, 100, 150, 299, 300][-M:])


@pytest.mark.parametrize("npig", [4, 8])
def test_accumulate_recall_levels_on_thresholds(npig):
    """rc = k / npig lands exactly on 0.25 / 0.5 / 0.75 / 1.0: searchsorted(side="left") takes the first equal level."""
    rng = np.random.default_rng(npig)
    n = 24
    records = (np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.uint64), np.zeros(n, np.uint64),
               np.array([[npig, npig, 0, 0]], np.int32))
    hits = rng.permutation(np.r_[np.ones(npig), np.zeros(n - npig)]).astype(np.uint64)
    records[2][:] = hits | (hits << np.uint64(1))
    score = np.linspace(1, 0.1, n).astype(np.float32)
    check_accumulate(records, score, 1, 1, [0.25, 0.5, 0.75, 1.0], [100])


# ---- K12: packing ------------------------------------------------------------------------------------------------------------
def pack_oracle(masks):
    n = masks.shape[0]
    flat = (masks.reshape(n, -1) != 0)
    hw = flat.shape[1]
    words = (hw + 31) // 32
    pad = np.zeros((n, words * 32), bool)
    pad[:, :hw] = flat
    return np.packbits(pad, axis=1, bitorder="little").view("<u4").reshape(n, words), flat.sum(1)


def pack_grid(n, hw):
    """mb200_mask_pack_bits: warps of 2048-pixel chunks, 8 per CTA, grid capped at sm_count * 8 (then the warps loop)."""
    return min((n * ((hw + 2047) // 2048) + 7) // 8, sm_count() * 8)


@pytest.mark.parametrize("hw", [1, 31, 33, 2047, 2048, 2049, 4095, 4096, 4097, 6143, 6144, 6145])
@pytest.mark.parametrize("offset", [0, 1])
def test_mask_pack(hw, offset):
    rng = np.random.default_rng(hw + offset)
    n = 5
    values = rng.choice(np.array([0, 0, 0, 1, 2, 128, 255], np.uint8), (n, hw))
    buf = torch.zeros(n * hw + 16, dtype=torch.uint8, device=DEV)
    buf[offset:offset + n * hw] = t(values.reshape(-1))
    masks = buf[offset:offset + n * hw].view(n, 1, hw)
    assert (masks.data_ptr() % 16 == 0) == (offset == 0)
    want_words, want_area = pack_oracle(values)
    words, area = _native.mask_pack_bits(masks)
    np.testing.assert_array_equal(words.cpu().numpy().view(np.uint32), want_words)
    np.testing.assert_array_equal(area.cpu().numpy(), want_area)
    entry = _native.mask_pack_entry(masks).cpu().numpy()
    assert entry[:3].tolist() == [n, 1, hw]
    np.testing.assert_array_equal(entry[3:3 + n], want_area)
    np.testing.assert_array_equal(entry[3 + n:].view(np.uint32), want_words.reshape(-1))


def test_mask_pack_grid_cap():
    n, hw = 9000, 40
    assert (n * 1 + 7) // 8 > sm_count() * 8 == pack_grid(n, hw)
    values = (np.random.default_rng(0).random((n, hw)) < 0.5).astype(np.uint8)
    words, area = _native.mask_pack_bits(t(values).view(n, 5, 8))
    want_words, want_area = pack_oracle(values)
    np.testing.assert_array_equal(words.cpu().numpy().view(np.uint32), want_words)
    np.testing.assert_array_equal(area.cpu().numpy(), want_area)
    entry = _native.mask_pack_entry(t(values).view(n, 5, 8)).cpu().numpy()
    np.testing.assert_array_equal(entry[3:3 + n], want_area)
    np.testing.assert_array_equal(entry[3 + n:].view(np.uint32), want_words.reshape(-1))


@pytest.mark.raw_abi
def test_mask_pack_output_stride_wider_than_a_row():
    n, hw, stride = 7, 3000, 101
    values = (np.random.default_rng(1).random((n, hw)) < 0.3).astype(np.uint8) * 9
    masks = t(values)
    out = torch.full((n, stride), -0x5A5A5A5B, dtype=torch.int32, device=DEV)
    area = torch.full((n,), 12345, dtype=torch.int64, device=DEV)
    rc = _native.lib().mb200_mask_pack_bits(masks.data_ptr(), n, hw, out.data_ptr(), stride, area.data_ptr(),
                                            _native.stream_handle(torch.device(DEV)))
    assert rc == 0
    want_words, want_area = pack_oracle(values)
    got = out.cpu().numpy()
    np.testing.assert_array_equal(got[:, :94].view(np.uint32), want_words)
    assert (got[:, 94:] == -0x5A5A5A5B).all()
    np.testing.assert_array_equal(area.cpu().numpy(), want_area)


def test_mask_pack_no_pixels():
    words, area = _native.mask_pack_bits(torch.zeros((3, 0, 5), dtype=torch.bool, device=DEV))
    assert tuple(words.shape) == (3, 0) and area.cpu().tolist() == [0, 0, 0]
    assert _native.mask_pack_entry(torch.zeros((3, 0, 5), dtype=torch.bool, device=DEV)).cpu().tolist() == [3, 0, 5, 0, 0, 0]


def test_mask_pack_more_than_2_32_bytes():
    """Two masks of 2^31 + 2049 pixels (4 GiB + 4098 bytes, the second row unaligned), striped: pixel p of mask m is 3
    where (p + 2 m) % 5 == 0.  Words at the first / last word and around the 2^31 / 2^32 byte offsets; both areas."""
    n, hw = 2, 2 ** 31 + 2049
    period = 5 * 4096
    stripe = torch.zeros(period, dtype=torch.uint8, device=DEV)
    masks = torch.empty((n, 1, hw), dtype=torch.uint8, device=DEV)
    for m in range(n):
        stripe.zero_()
        stripe[(-2 * m) % 5::5] = 3
        reps = hw // period
        masks[m, 0, :reps * period].view(reps, period).copy_(stripe.expand(reps, period))
        masks[m, 0, reps * period:] = stripe[:hw - reps * period]
    words, area = _native.mask_pack_bits(masks)
    words = words.cpu().numpy().view(np.uint32)
    nw = (hw + 31) // 32

    def want_word(m, w):
        return sum(1 << k for k in range(32) if 32 * w + k < hw and (32 * w + k + 2 * m) % 5 == 0)

    for m in range(n):
        assert int(area[m]) == len(range((-2 * m) % 5, hw, 5))
    probe = {(0, 0), (0, 1), (n - 1, nw - 1), (n - 1, nw - 2)}
    for byte in (2 ** 31, 2 ** 32):
        m, p = divmod(byte, hw)
        for w in (p // 32 - 1, p // 32, p // 32 + 1):
            if 0 <= w < nw:
                probe.add((m, w))
    for m, w in sorted(probe):
        assert int(words[m, w]) == want_word(m, w), (m, w)


# ---- K12: pair intersections --------------------------------------------------------------------------------------------------
def pair_splits(n_img, max_pairs):
    splits = (max_pairs // 8 + 1 + 7) // 8
    want = (sm_count() * 8 + n_img - 1) // n_img
    return max(1, min(splits, want, 65535)), splits > want


def run_pairs(seed, shapes, micro=False, n_labels=3):
    """`shapes`: per image (D, G, words)."""
    rng = np.random.default_rng(seed)
    det_rows, gt_rows, det_lab, gt_lab = [], [], [], []
    for d, g, w in shapes:
        det_rows += [rng.integers(0, 2 ** 32, w, dtype=np.uint64).astype(np.uint32) & rng.integers(0, 2 ** 32, w, dtype=np.uint64).astype(np.uint32) for _ in range(d)]
        gt_rows += [rng.integers(0, 2 ** 32, w, dtype=np.uint64).astype(np.uint32) for _ in range(g)]
        det_lab += rng.integers(0, n_labels, d).tolist()
        gt_lab += rng.integers(0, n_labels, g).tolist()
    flat = lambda rows: np.concatenate(rows + [np.zeros(1, np.uint32)])  # noqa: E731
    off = lambda rows: np.concatenate([[0], np.cumsum([len(r) for r in rows])[:-1]]).astype(np.int64) if rows else np.zeros(0, np.int64)  # noqa: E731
    det_off = np.concatenate([[0], np.cumsum([s[0] for s in shapes])]).astype(np.int32)
    gt_off = np.concatenate([[0], np.cumsum([s[1] for s in shapes])]).astype(np.int32)
    sizes = [d * g for d, g, _ in shapes]
    pair_off = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    n_pairs, max_pairs = int(sum(sizes)), max(sizes)
    got = _native.mask_pair_intersections(
        t(flat(det_rows).view(np.int32)), t(off(det_rows)), t(flat(gt_rows).view(np.int32)), t(off(gt_rows)), t(det_off),
        t(gt_off), t(np.array([s[2] for s in shapes], np.int32)), t(np.array(det_lab, np.int64)), t(np.array(gt_lab, np.int64)),
        micro, t(pair_off), n_pairs, max_pairs).cpu().numpy()
    for i, (d, g, w) in enumerate(shapes):
        if d == 0 or g == 0:
            continue
        a = np.stack(det_rows[det_off[i]:det_off[i + 1]])
        b = np.stack(gt_rows[gt_off[i]:gt_off[i + 1]])
        inter = np.unpackbits((a[:, None, :] & b[None, :, :]).view(np.uint8), axis=2).sum(2).astype(np.float64)
        if not micro:
            same = np.array(det_lab[det_off[i]:det_off[i + 1]])[:, None] == np.array(gt_lab[gt_off[i]:gt_off[i + 1]])[None, :]
            inter = np.where(same, inter, 0.0)
        np.testing.assert_array_equal(got[pair_off[i]:pair_off[i] + d * g].reshape(d, g), inter, err_msg=f"image {i}")
    return pair_splits(len(shapes), max_pairs)


@pytest.mark.parametrize("micro", [False, True])
def test_mask_pairs_every_tile_remainder(micro):
    shapes = [(d, g, 33 + 7 * ((d * 9 + g) % 5)) for d in range(1, 10) for g in range(1, 10)]
    shapes[3] = (0, 4, 40)
    shapes[10] = (5, 0, 40)
    run_pairs(1, shapes, micro=micro)


def test_mask_pairs_label_mismatch_is_zero():
    run_pairs(2, [(6, 7, 50), (3, 3, 64)], n_labels=2)


def test_mask_pairs_several_ctas_per_image():
    splits, capped = run_pairs(3, [(60, 45, 70), (9, 0, 33), (17, 13, 90)])
    assert splits > 1 and not capped


def test_mask_pairs_split_count_capped_by_image_count():
    shapes = [(int(d), int(g), 33 + i % 40) for i, (d, g) in enumerate(np.random.default_rng(4).integers(1, 10, (2000, 2)))]
    shapes[0] = (40, 40, 35)
    splits, capped = run_pairs(4, shapes, micro=False)
    assert capped and splits == 1
