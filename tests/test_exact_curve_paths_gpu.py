"""GPU: exact-mode curve evaluation (K3 / K5: csrc/curve.cu, csrc/radix_sort.cuh) against the reference's chain restated in
torch (oracle/exact_curves.py) on the same GPU, on every entry point and launch path:
  entry     pair keys (`mb200_curve_evaluate`), label in bit 0 (`_nonneg`, and `unit_range=None` with its fall-back on a
            negative score), multilabel with and without `ignore_index`, pre-packed keys (`_keys` / `_keys_nonneg` with
            first_class > 0), the weighted curve
  dtypes    float32 / float16 / bfloat16 scores (4 radix passes), float64 (8 passes, no bit-0 path); targets of every
            integer dtype and bool, on both sides of the int64 pack instantiation
  geometry  n on both sides of the radix tile (8192) and the scan tile (4096); more than 9 sort tiles (a second look-back
            window); more than 33 scan tiles (a second 32-wide look-back round) and more than 256 (the wide finalize);
            n % 4 != 0 with several segments (scalar scan loads); n and C not multiples of 32 (the transpose tiles); the
            binary pack's grid-stride loop; 1, 2, 33, 1000 and 65535 segments (the histogram grid cap), and the errors for
            65536 segments and n = 2^30; one binary case at n = 2^30 - 1
  values    every float16 / bfloat16 bit pattern (each NaN payload, +-0, subnormals, +-inf), NaN runs crossing tile
            boundaries, ties longer than a tile, all-positive and all-negative segments, a workspace holding stale bytes
Every case first asserts its path with `path_of`, a restatement of the dispatch in `evaluate_typed`, `sort_and_scan` and
`radix_sort_passes*`, runs the kernel twice on one workspace with the error word zero after each run, and requires
`torch.equal` on counts, fps, tps and thresholds, and on the bits of AUROC, against the oracle; AP within one float32 ulp of
its float64 value (the kernel divides with a refined hardware reciprocal).  Where a NaN / +-inf run holds both labels the
oracle takes the documented order (negatives before positives inside the run), elsewhere the reference's own argsort.
"""
import ctypes

import pytest
import torch

from metrics_b200 import _native
from oracle import exact_curves as oe

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F16, BF16, F32, F64 = torch.float16, torch.bfloat16, torch.float32, torch.float64
INT_TARGETS = [torch.int64, torch.int32, torch.int16, torch.int8, torch.uint8, torch.bool]
SORT_TILE, SCAN_TILE, PACK_STRIDE = 8192, 4096, 132 * 8 * 1024
NAN, INF = float("nan"), float("inf")


# ------------------------------------------------------------------------------------------------------------------
# the dispatch of curve.cu / radix_sort.cuh, restated
# ------------------------------------------------------------------------------------------------------------------
def sm_count():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def path_of(entry, dtype, n, segments, target_dtype=torch.int64):
    """The launch path as a dict: keys (pair / bit0), radix passes, pack kernel, pack grid-stride rounds (binary pack),
    sort tiles per segment, histogram grid (counted by the pack / full / capped at sm_count*8/segments), scan tiles per
    segment, finalize (warp / wide) and the scan loads of segments after the first (vector when their records stay 16-byte
    aligned, scalar when n % 16 != 0).  `nonneg` is the label-in-bit-0 entry, which float64 scores (8-byte keys) leave for
    the pair path.  Every case compares it with literal expectations (`expect`)."""
    if entry in ("keys", "keys_nonneg"):
        bit0, pack = entry == "keys_nonneg", "keys"
    elif entry == "multilabel":
        bit0, pack = False, "multilabel"
    elif entry == "weighted":
        bit0, pack = False, "indexed"
    else:
        bit0 = entry == "nonneg" and dtype != F64
        pack = ("binary" if segments == 1 else "ovr") + ("_i64" if segments == 1 and target_dtype == torch.int64 else "")
    passes = 8 if dtype == F64 else 4
    sort_tiles = -(-n // SORT_TILE)
    hcap = max(1, sm_count() * 8 // segments)
    hist = "pack" if bit0 and pack.startswith("binary") else ("capped" if -(-n // 4096) > hcap else "full")
    scan_tiles = -(-n // SCAN_TILE)
    pack_grid = min(-(-n // 1024), sm_count() * 8)
    return dict(keys="bit0" if bit0 else "pair", passes=passes, pack=pack,
                pack_rounds=-(-n // (pack_grid * 1024)) if pack.startswith("binary") else 1, sort_tiles=sort_tiles,
                hist=hist, scan_tiles=scan_tiles, finalize="wide" if scan_tiles > 256 else "warp",
                seg_load="single" if segments == 1 else ("vector" if n % 16 == 0 else "scalar"))


def expect(path, want):
    """Each field of `want` is a literal or a predicate on the field."""
    for k, v in want.items():
        assert (v(path[k]) if callable(v) else path[k] == v), (k, path[k], v, path)


# ------------------------------------------------------------------------------------------------------------------
# the C-ABI with an error word and a caller-owned workspace
# ------------------------------------------------------------------------------------------------------------------
P, I64 = _native.ptr, _native.i64


def stale_workspace(nbytes):
    g = torch.Generator(device=DEV).manual_seed(nbytes % 1000)
    return torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device=DEV, generator=g)


def evaluate(entry, preds, target, segments, pos_label=1, ignore_index=None, first_class=0, want_curve=True, want_err=0):
    """Runs the entry twice on one workspace (stale random bytes the first time, the first run's the second); both runs
    must agree and leave the error word at `want_err` (zero: no range flag, no look-back timeout).
    Returns (auroc, ap, counts, curve)."""
    lib = _native.lib()
    keys_mode = entry in ("keys", "keys_nonneg")
    n = preds.shape[0]
    if keys_mode:
        nbytes = int(lib.mb200_curve_workspace_bytes(I64(segments), I64(n)))
    else:
        nbytes = int(lib.mb200_curve_workspace_bytes_for(I64(segments), I64(n), _native.tag(preds)))
    ws = stale_workspace(nbytes)
    st = _native.stream_handle(torch.device(DEV))
    results = []
    for _ in range(2):
        err = torch.zeros(1, dtype=torch.int32, device=DEV)
        auroc = torch.empty(segments, dtype=F32, device=DEV)
        ap = torch.empty(segments, dtype=F32, device=DEV)
        counts = torch.empty((segments, 3), dtype=torch.int64, device=DEV)
        curve = None
        if want_curve and not keys_mode:
            thr_dt = F64 if preds.dtype == F64 else F32
            curve = tuple(torch.full((segments, n), 7.0, dtype=dt, device=DEV) for dt in (F32, F32, thr_dt))
        c3 = (P(curve[0]), P(curve[1]), P(curve[2])) if curve else (None, None, None)
        if entry in ("pair", "nonneg"):
            fn = lib.mb200_curve_evaluate_nonneg if entry == "nonneg" else lib.mb200_curve_evaluate
            rc = fn(P(preds), _native.tag(preds), P(target), _native.tag(target), I64(n), I64(segments), I64(pos_label),
                    P(ws), I64(nbytes), P(auroc), P(ap), P(counts), *c3, P(err), st)
        elif entry == "multilabel":
            rc = lib.mb200_curve_evaluate_multilabel(
                P(preds), _native.tag(preds), P(target), _native.tag(target), I64(n), I64(segments),
                ctypes.c_int(0 if ignore_index is None else 1), I64(0 if ignore_index is None else ignore_index), P(ws),
                I64(nbytes), P(auroc), P(ap), P(counts), *c3, P(err), st)
        else:
            keys = _native.curve_pack_keys(preds)
            fn = lib.mb200_curve_evaluate_keys_nonneg if entry == "keys_nonneg" else lib.mb200_curve_evaluate_keys
            rc = fn(P(keys), P(target), _native.tag(target), I64(n), I64(segments), I64(first_class), P(ws), I64(nbytes),
                    P(auroc), P(ap), P(counts), P(err), st)
        _native.check(rc, entry)
        torch.cuda.synchronize()
        assert int(err) == want_err, f"error word {int(err)} after {entry}"
        results.append((auroc, ap, counts, curve))
    (a0, p0, c0, k0), (a1, p1, c1, k1) = results
    assert torch.equal(a0, a1) and torch.equal(p0, p1) and torch.equal(c0, c1)
    if k0:
        assert all(same(x, y) for x, y in zip(k0, k1))
    return results[1]


# ------------------------------------------------------------------------------------------------------------------
# comparison with the oracle
# ------------------------------------------------------------------------------------------------------------------
def mixed_special_run(p, positive):
    """A NaN / +inf / -inf run holding both labels: only the documented order pins the result."""
    p = p.double()
    for m in (p.isnan(), p == INF, p == -INF):
        if bool((m & positive).any()) and bool((m & ~positive).any()):
            return True
    return False


def same(a, b):
    return a.shape == b.shape and torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(3.0), b.nan_to_num(3.0))


def f32_ulp_close(got, want):
    w = torch.tensor(want, dtype=F32)
    return float(got) == float(w) or abs(float(got) - float(w)) <= float(torch.nextafter(w.abs(), torch.tensor(INF)) - w.abs())


def check_segment(s, p, t, pos_label, auroc, ap, counts, curve, info, weights=None):
    positive = t == pos_label
    documented = mixed_special_run(p, positive)
    fps, tps, thr = oe.binary_clf_curve(p, t, pos_label=pos_label, documented_order=documented)
    U = thr.numel()
    Pn = int(positive.sum())
    assert counts[s].tolist() == [Pn, p.numel() - Pn, U], (info, s, counts[s].tolist(), [Pn, p.numel() - Pn, U])
    if curve is not None:
        assert torch.equal(curve[0][s, :U], fps.float()), (info, s, "fps")
        assert torch.equal(curve[1][s, :U], tps.float()), (info, s, "tps")
        want_thr = thr.double() if p.dtype == F64 else thr.float()
        assert same(curve[2][s, :U], want_thr), (info, s, "thresholds")
    want_auc = oe.auroc_exact(fps.long(), tps.long())
    assert float(auroc[s]) == float(torch.tensor(want_auc, dtype=F32)), (info, s, float(auroc[s]), want_auc)
    want_ap = oe.average_precision_exact(fps.long(), tps.long())
    assert f32_ulp_close(ap[s], want_ap), (info, s, float(ap[s]), want_ap)


def check_binary(entry, p, t, pos_label=1, want_path=None, want_curve=True):
    if want_path is not None:
        expect(path_of(entry, p.dtype, p.numel(), 1, t.dtype), want_path)
    auroc, ap, counts, curve = evaluate(entry, p, t, 1, pos_label, want_curve=want_curve)
    check_segment(0, p, t, pos_label, auroc, ap, counts, curve, (entry, p.dtype, t.dtype, p.numel()))


def check_ovr(entry, p, t, first_class=0, sample=None, want_path=None):
    n, C = p.shape
    if want_path is not None:
        expect(path_of(entry, p.dtype, n, C), want_path)
    auroc, ap, counts, curve = evaluate(entry, p, t, C, first_class=first_class)
    for s in (range(C) if sample is None else sample):
        check_segment(s, p[:, s], t, first_class + s, auroc, ap, counts, curve, (entry, p.dtype, t.dtype, n, C))


def check_multilabel(p, t, ignore_index=None, want_path=None):
    n, L = p.shape
    if want_path is not None:
        expect(path_of("multilabel", p.dtype, n, L), want_path)
    auroc, ap, counts, curve = evaluate("multilabel", p, t, L, ignore_index=ignore_index)
    for s, (ps, ts) in enumerate(oe.multilabel_columns(p, t, L, ignore_index)):
        check_segment(s, ps, ts, 1, auroc, ap, counts, curve, ("multilabel", p.dtype, t.dtype, n, L, ignore_index))


# ------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------
def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def scores(shape, dtype, seed, levels=None, nan_frac=0.0, inf=False):
    g = gen(seed)
    x = torch.rand(shape, generator=g, device=DEV, dtype=F64)
    if levels:
        x = torch.floor(x * levels) / levels  # long tie runs
    if nan_frac:
        x[torch.rand(shape, generator=g, device=DEV) < nan_frac] = NAN
    if inf:
        r = torch.rand(shape, generator=g, device=DEV)
        x[r < 0.01] = INF
    return x.to(dtype)


def labels(shape, dtype, seed, high=2):
    shape = (shape,) if isinstance(shape, int) else shape
    t = torch.randint(0, high, shape, generator=gen(seed + 1), device=DEV)
    return t.bool() if dtype == torch.bool else t.to(dtype)


# (n, sort tiles, scan tiles, finalize): both sides of the scan tile (4096) and the radix tile (8192), > 9 sort tiles (a
# second look-back window of 8), > 33 scan tiles (a second 32-wide look-back round), > 256 scan tiles (the wide finalize)
SIZES = [(1, 1, 1, "warp"), (31, 1, 1, "warp"), (4095, 1, 1, "warp"), (4096, 1, 1, "warp"), (4097, 1, 2, "warp"),
         (8191, 1, 2, "warp"), (8192, 1, 2, "warp"), (8193, 2, 3, "warp"), (73733, 10, 19, "warp"),
         (135171, 17, 34, "warp"), (1052685, 129, 258, "wide")]


# ------------------------------------------------------------------------------------------------------------------
# binary: pair and bit-0 entries, every geometry
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,sort_tiles,scan_tiles,finalize", SIZES)
@pytest.mark.parametrize("dtype", [F32, F64])
def test_pair_geometry(n, sort_tiles, scan_tiles, finalize, dtype):
    p, t = scores(n, dtype, n, levels=3000, nan_frac=0.02), labels(n, torch.int64, n)
    check_binary("pair", p, t, want_path=dict(keys="pair", passes=8 if dtype == F64 else 4, pack="binary_i64", hist="full",
                                              sort_tiles=sort_tiles, scan_tiles=scan_tiles, finalize=finalize))


@pytest.mark.parametrize("n,sort_tiles,scan_tiles,finalize", SIZES)
def test_bit0_geometry(n, sort_tiles, scan_tiles, finalize):
    p, t = scores(n, F32, n + 5, levels=3000, nan_frac=0.02), labels(n, torch.int32, n + 5)
    check_binary("nonneg", p, t, want_path=dict(keys="bit0", passes=4, pack="binary", hist="pack", sort_tiles=sort_tiles,
                                                scan_tiles=scan_tiles, finalize=finalize))


def test_pack_grid_stride_loop():
    n = PACK_STRIDE * 2 + 7
    p, t = scores(n, F16, 3, nan_frac=0.001, inf=True), labels(n, torch.uint8, 3)
    want = dict(pack="binary", pack_rounds=lambda r: r >= 2, scan_tiles=529, finalize="wide")
    check_binary("pair", p, t, want_path=dict(want, keys="pair"))
    check_binary("nonneg", p.abs(), t, want_path=dict(want, keys="bit0"))


@pytest.mark.parametrize("tdt", INT_TARGETS)
@pytest.mark.parametrize("dtype", [F32, F16, BF16, F64])
def test_target_dtypes(dtype, tdt):
    n = 3 * SCAN_TILE + 3
    p, t = scores(n, dtype, 11, levels=500, nan_frac=0.05), labels(n, tdt, 11)
    want = dict(pack="binary_i64" if tdt == torch.int64 else "binary", passes=8 if dtype == F64 else 4, sort_tiles=2,
                scan_tiles=4)
    check_binary("pair", p, t, want_path=dict(want, keys="pair"))
    if dtype != F64:
        check_binary("nonneg", p, t, want_path=dict(want, keys="bit0"))


def test_int64_targets_beyond_int32():
    n = 5000
    t = labels(n, torch.int64, 5) * (2**32 + 1)  # 2^32 + 1 is not label 1
    t[::7] = 2**31
    t[::11] = 1
    p = scores(n, F32, 5, nan_frac=0.03)
    check_binary("pair", p, t)
    check_binary("nonneg", p, t)


@pytest.mark.parametrize("entry", ["pair", "nonneg"])
def test_ovr_int64_targets_beyond_int32(entry):
    n, C = 5000, 3
    p, t = scores((n, C), F32, 6), labels(n, torch.int64, 6, high=C)  # finite scores: only the target compare differs
    t[::5] += 2**32  # 2^32 + c is no class
    check_ovr(entry, p, t, want_path=dict(pack="ovr", scan_tiles=2, seg_load="scalar"))


@pytest.mark.parametrize("dtype", [F16, BF16])
def test_every_half_bit_pattern(dtype):
    bits = torch.arange(-(2**15), 2**15, dtype=torch.int32, device=DEV).to(torch.int16)
    p = bits.view(dtype)
    for seed in (0, 1):
        t = labels(p.numel(), torch.int64, seed)
        check_binary("pair", p, t)
        check_binary("pair", p.float(), t)
        nonneg = p[bits >= 0]  # +0 .. +NaN payloads: the bit-0 path
        check_binary("nonneg", nonneg, t[: nonneg.numel()])


def test_unit_range_none_falls_back_on_a_negative_score():
    n = 20000
    p, t = scores(n, F32, 9, nan_frac=0.05), labels(n, torch.int64, 9)
    p[n // 2] = -0.25
    # the bit-0 attempt raises the range flag, which is what sends unit_range=None back to the pair path
    evaluate("nonneg", p, t, 1, want_curve=False, want_err=2)
    auroc, ap, counts, curve = _native.curve_evaluate(p, t, 1, want_curve=True, unit_range=None)
    check_segment(0, p, t, 1, auroc, ap, counts, curve, "unit_range=None")
    p[n // 2] = -0.0  # -0 stays on the bit-0 path
    evaluate("nonneg", p, t, 1)  # error word zero
    auroc, ap, counts, curve = _native.curve_evaluate(p, t, 1, want_curve=True, unit_range=None)
    check_segment(0, p, t, 1, auroc, ap, counts, curve, "unit_range=None, -0")


@pytest.mark.parametrize("entry", ["pair", "nonneg"])
def test_special_runs_across_tiles(entry):
    """NaN / +inf runs of mixed labels longer than a scan tile and straddling sort and scan tile boundaries, and a tie run
    longer than a sort tile; -inf runs on the pair path."""
    n = 5 * SORT_TILE + 77
    p = scores(n, F32, 21, levels=40)
    p[: SORT_TILE + 100] = NAN
    p[2 * SORT_TILE - 50: 3 * SORT_TILE + 50] = INF
    p[3 * SORT_TILE + 50: 4 * SORT_TILE + 3000] = 0.5
    if entry == "pair":
        p[-SCAN_TILE - 9:] = -INF
    t = labels(n, torch.int64, 21)
    perm = torch.randperm(n, generator=gen(22), device=DEV)
    check_binary(entry, p[perm].contiguous(), t)


@pytest.mark.parametrize("entry", ["pair", "nonneg"])
@pytest.mark.parametrize("label", [0, 1])
def test_single_class_segments(entry, label):
    n = 2 * SCAN_TILE + 1
    p = scores(n, F32, 31, levels=100, nan_frac=0.1)
    t = torch.full((n,), label, dtype=torch.int64, device=DEV)
    check_binary(entry, p, t)


# ------------------------------------------------------------------------------------------------------------------
# one-vs-rest, multilabel, pre-packed keys
# ------------------------------------------------------------------------------------------------------------------
# (n, C, sort tiles, scan tiles, histogram grid, later segments' scan loads); "capped": ceil(n / 4096) > sm_count * 8 / C
OVR = [(4099, 3, 1, 2, "full", "scalar"), (33, 33, 1, 1, "full", "scalar"), (8198, 2, 2, 3, "full", "scalar"),
       (97, 1000, 1, 1, "full", "scalar"), (5001, 33, 1, 2, "full", "scalar"), (8193, 1000, 2, 3, "capped", "scalar"),
       (200000, 33, 25, 49, "capped", "vector")]


@pytest.mark.parametrize("n,C,sort_tiles,scan_tiles,hist,seg_load", OVR)
@pytest.mark.parametrize("entry", ["pair", "nonneg"])
def test_ovr_geometry(entry, n, C, sort_tiles, scan_tiles, hist, seg_load):
    p, t = scores((n, C), F32, n + C, levels=200, nan_frac=0.05), labels(n, torch.int64, n + C, high=C)
    sample = None if C <= 33 else list(range(0, C, 97)) + [C - 1]
    check_ovr(entry, p, t, sample=sample, want_path=dict(keys="bit0" if entry == "nonneg" else "pair", pack="ovr",
                                                         sort_tiles=sort_tiles, scan_tiles=scan_tiles, hist=hist,
                                                         seg_load=seg_load))


@pytest.mark.parametrize("dtype", [F16, BF16])
def test_ovr_bit0_half_scores(dtype):
    n, C = 4101, 7
    p = scores((n, C), dtype, 43, levels=300, nan_frac=0.05, inf=True)
    check_ovr("nonneg", p, labels(n, torch.int32, 43, high=C), want_path=dict(keys="bit0", pack="ovr", seg_load="scalar"))


def test_ovr_f64_and_half_targets():
    n, C = 4101, 5
    for dtype in (F64, BF16):
        for tdt in (torch.uint8, torch.int16, torch.bool):
            high = 2 if tdt == torch.bool else C
            check_ovr("pair", scores((n, C), dtype, 41, nan_frac=0.05, inf=True), labels(n, tdt, 41, high=high),
                      want_path=dict(keys="pair", passes=8 if dtype == F64 else 4, pack="ovr", scan_tiles=2))


def test_segment_limit_and_errors():
    n, C = 3, 65535
    p, t = scores((n, C), F32, 51, nan_frac=0.2), labels(n, torch.int64, 51, high=C)
    t[0] = C - 1
    check_ovr("pair", p, t, sample=[0, 1, 2, C // 2, C - 1],
              want_path=dict(pack="ovr", sort_tiles=1, scan_tiles=1, hist="full", seg_load="scalar"))
    lib = _native.lib()
    buf = torch.zeros(64, dtype=torch.uint8, device=DEV)
    out = torch.zeros(64, dtype=torch.int64, device=DEV)
    st = _native.stream_handle(torch.device(DEV))
    # both refusals return before any launch (size checks come first), so the small buffers are never read
    for n_, C_, wsb in ((2**30, 1, 1 << 62), (4, 65536, 1 << 62)):
        rc = lib.mb200_curve_evaluate(P(buf), _native.tag(p), P(buf), _native.tag(t), I64(n_), I64(C_), I64(1), P(buf),
                                      I64(wsb), P(buf), P(buf), P(out), None, None, None, None, st)
        assert rc != 0, (n_, C_)


@pytest.mark.parametrize("tdt,ign,vals", [
    (torch.uint8, 257, [0, 1, 255]), (torch.uint8, -1, [0, 1, 255]), (torch.int8, 255, [0, 1, -1]),
    (torch.int16, 65535, [0, 1, -1]), (torch.int64, -1, [0, 1, -1]), (torch.int32, None, [0, 1, 2]),
    (torch.bool, 0, [False, True]), (torch.bool, -1, [False, True]),  # bool targets: the value is not wrapped
])
@pytest.mark.parametrize("dtype", [F32, F64])
def test_multilabel_wrapped_ignore_index(dtype, tdt, ign, vals):
    n, L = 4101, 37
    p = scores((n, L), dtype, 61, levels=300, nan_frac=0.05, inf=True)
    idx = torch.randint(0, len(vals), (n, L), generator=gen(62), device=DEV)
    t = torch.tensor(vals, device=DEV)[idx].to(tdt)
    check_multilabel(p, t, ign, want_path=dict(pack="multilabel", passes=8 if dtype == F64 else 4, sort_tiles=1,
                                               scan_tiles=2, seg_load="scalar"))


@pytest.mark.parametrize("entry", ["keys", "keys_nonneg"])
@pytest.mark.parametrize("n,S,first,sort_tiles,scan_tiles", [(4099, 3, 2, 1, 2), (SORT_TILE + 3, 2, 5, 2, 3),
                                                             (37, 33, 1, 1, 1)])
def test_packed_keys(entry, n, S, first, sort_tiles, scan_tiles):
    p = scores((n, S), F32, n + S, levels=100, nan_frac=0.05, inf=True)  # +inf reaches fold_labels_into_keys too
    t = labels(n, torch.int64, n + S, high=S + first)
    check_ovr(entry, p, t, first_class=first, want_path=dict(keys="bit0" if entry == "keys_nonneg" else "pair", pack="keys",
                                                             sort_tiles=sort_tiles, scan_tiles=scan_tiles,
                                                             seg_load="scalar"))


@pytest.mark.parametrize("dtype", [F32, F64])
def test_weighted_curve(dtype):
    n = 3 * 1024 + 5
    p = scores(n, dtype, 71, levels=50, nan_frac=0.05, inf=True)
    p[::13] = -INF
    t = labels(n, torch.int64, 71)
    w = torch.randint(1, 6, (n,), generator=gen(72), device=DEV).double()  # integer weights: exact sums in any order
    fps, tps, thr = _native.curve_weighted_clf_curve(p, t, w)
    wf, wt, wthr = oe.binary_clf_curve(p, t, sample_weights=w, documented_order=True)
    assert torch.equal(fps, wf) and torch.equal(tps, wt)
    assert same(thr, wthr.double() if dtype == F64 else wthr.float())


# ------------------------------------------------------------------------------------------------------------------
# public surface
# ------------------------------------------------------------------------------------------------------------------
def test_functionals_and_classes_with_nan_runs_and_wrapped_ignore():
    import metrics_b200.classification as mc
    import metrics_b200.functional.classification as fc

    n = 3000
    p, t = scores(n, F32, 81, nan_frac=0.05), labels(n, torch.int64, 81)
    fp, ft = oe.binary_format(p, t)
    fps, tps, thr = oe.binary_clf_curve(fp, ft, documented_order=True)
    for got, want in zip(fc.binary_roc(p, t, validate_args=False), oe.binary_roc(fps, tps, thr)):
        assert same(got, want)
    for got, want in zip(fc.binary_precision_recall_curve(p, t, validate_args=False), oe.binary_pr(fps, tps, thr, ft)):
        assert same(got, want)
    auc = oe.auroc_exact(fps.long(), tps.long())
    assert float(fc.binary_auroc(p, t, validate_args=False)) == pytest.approx(auc, rel=2e-6)
    m = mc.BinaryAUROC(validate_args=False).to(DEV)
    m.update(p[: n // 2], t[: n // 2])
    m.update(p[n // 2:], t[n // 2:])
    assert float(m.compute()) == pytest.approx(auc, rel=2e-6)

    L = 3
    pm = scores((n, L), F32, 82, nan_frac=0.05)
    tm = torch.tensor([0, 1, 255], dtype=torch.uint8, device=DEV)[torch.randint(0, 3, (n, L), generator=gen(83), device=DEV)]
    cols = oe.multilabel_columns(*oe.multilabel_format(pm, tm, L), L, -1)  # -1 is 255 in uint8
    got = fc.multilabel_auroc(pm, tm, num_labels=L, average="none", ignore_index=-1, validate_args=False)
    for i, (ps, ts) in enumerate(cols):
        f, tp_, _ = oe.binary_clf_curve(ps, ts, documented_order=True)
        assert float(got[i]) == pytest.approx(oe.auroc_exact(f.long(), tp_.long()), rel=2e-6), i
    ma = mc.MultilabelAveragePrecision(num_labels=L, average="none", ignore_index=-1, validate_args=False).to(DEV)
    ma.update(pm, tm)
    got = ma.compute()
    roc = fc.multilabel_roc(pm, tm, num_labels=L, ignore_index=-1, validate_args=False)
    prc = fc.multilabel_precision_recall_curve(pm, tm, num_labels=L, ignore_index=-1, validate_args=False)
    for i, (ps, ts) in enumerate(cols):
        f, tp_, th = oe.binary_clf_curve(ps, ts, documented_order=True)
        assert float(got[i]) == pytest.approx(float(oe.binary_average_precision(f, tp_, th, ts)), rel=2e-6, nan_ok=True), i
        for k, want in enumerate(oe.binary_roc(f, tp_, th)):
            assert same(roc[k][i], want), ("multilabel_roc", i, k)
        for k, want in enumerate(oe.binary_pr(f, tp_, th, ts)):
            assert same(prc[k][i], want), ("multilabel_precision_recall_curve", i, k)

    C = 4
    pc = scores((n, C), F32, 84, nan_frac=0.05)
    tc = labels(n, torch.int64, 84, high=C)
    fmt_p, fmt_t = oe.multiclass_format(pc, tc, C)
    got = fc.multiclass_auroc(pc, tc, num_classes=C, average="none", validate_args=False)
    m = mc.MulticlassAveragePrecision(num_classes=C, average="none", validate_args=False).to(DEV)
    m.update(pc[: n // 2], tc[: n // 2])
    m.update(pc[n // 2:], tc[n // 2:])
    got_ap = m.compute()
    roc = fc.multiclass_roc(pc, tc, num_classes=C, validate_args=False)
    for c in range(C):
        f, tp_, th = oe.binary_clf_curve(fmt_p[:, c], fmt_t, pos_label=c, documented_order=True)
        assert float(got[c]) == pytest.approx(oe.auroc_exact(f.long(), tp_.long()), rel=2e-6), c
        assert float(got_ap[c]) == pytest.approx(float(oe.binary_average_precision(f, tp_, th, fmt_t == c)), rel=2e-6), c
        for k, want in enumerate(oe.binary_roc(f, tp_, th)):
            assert same(roc[k][c], want), ("multiclass_roc", c, k)


@pytest.mark.parametrize("dtype", [F16, BF16])
def test_torch_cuda_sort_puts_sign_set_half_nans_last(dtype):
    """The deviation DESIGN §3 records: over all 65 536 bit patterns, the reference's argsort on the GPU puts the NaNs with
    the sign bit set behind -inf, where the kernels, torch.sort's documentation and its CPU sort put every NaN first."""
    bits = torch.arange(-(2**15), 2**15, dtype=torch.int32).to(torch.int16)
    x = bits.view(dtype)
    neg_nan = x.isnan() & (bits < 0)
    k = int(neg_nan.sum())
    order = torch.argsort(x.to(DEV), descending=True, stable=True).cpu()
    assert bool(neg_nan[order[-k:]].all()) and not bool(neg_nan[order[:-k]].any())
    order = torch.argsort(x, descending=True, stable=True)
    assert bool(x[order[: int(x.isnan().sum())]].isnan().all())


# ------------------------------------------------------------------------------------------------------------------
# n = 2^30 - 1
# ------------------------------------------------------------------------------------------------------------------
def test_largest_binary_batch():
    n = 2**30 - 1
    free, _ = torch.cuda.mem_get_info(DEV)
    if free < 24 * 2**30:
        pytest.skip(f"needs about 24 GB free on the device ({free / 2**30:.1f} GB)")
    codes = torch.randint(0, 2**16, (n,), generator=gen(91), device=DEV, dtype=torch.int32)
    p = (65535 - codes).float() / 65536  # exact, strictly decreasing in the code
    del codes
    t = torch.randint(0, 2, (n,), generator=gen(92), device=DEV, dtype=torch.uint8)
    expect(path_of("pair", F32, n, 1, torch.uint8), dict(keys="pair", passes=4, pack="binary", sort_tiles=131072,
                                                          hist="capped", scan_tiles=262144, finalize="wide"))
    auroc, ap, counts, _ = evaluate("pair", p, t, 1, want_curve=False)
    codes = (65535 - p * 65536).int()
    fps, tps = oe.grouped_counts(codes, t.bool(), 2**16)
    del codes
    assert counts[0].tolist() == [int(tps[-1]), int(fps[-1]), fps.numel()]
    assert float(auroc[0]) == float(torch.tensor(oe.auroc_exact(fps, tps), dtype=F32))
    assert f32_ulp_close(ap[0], oe.average_precision_exact(fps, tps))
