"""CPU: the C-ABI of every include/metrics_b200*.h against its ctypes binding `_native.SIGNATURES`.

The headers are found by glob and parsed; the union of their declarations must be the table, the library must export and
bind it, and the Python mirrors of header constants must hold the header's values.  Every wrapper of `_native.py` is driven
once against REAL ctypes function pointers with the declared signatures, and once against the real library up to its first
CUDA call, so an argument-count or C-type slip fails without a GPU."""
import ctypes
import glob
import os
import re

import pytest
import torch

from metrics_b200 import _native
from tests.conftest import ROOT

HEADERS = sorted(glob.glob(os.path.join(ROOT, "include", "metrics_b200*.h")))
MAIN_HEADER = os.path.join(ROOT, "include", "metrics_b200.h")
STREAM = 0xABCD


def _source(path):
    """The header without its comments."""
    text = re.sub(r"/\*.*?\*/", "", open(path).read(), flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def _letter(ctype: str) -> str:
    """The `_native._C_TYPES` letter of a C type: p void*/T*, s const char*, i int, q int64_t, Q uint64_t, d double."""
    if "*" in ctype:
        return "s" if "char" in ctype else "p"
    return {"int": "i", "int64_t": "q", "uint64_t": "Q", "double": "d"}[ctype.replace("const", "").split()[0]]


def _header_signatures(path):
    """{name: (return letter, argument letters)} of every entry point declared in one header."""
    out = {}
    for ret, name, args in re.findall(r"MB200_API\s+([\w\s\*]+?)\s*(mb200_\w+)\s*\(([^)]*)\)\s*;", _source(path)):
        params = [a.strip() for a in " ".join(args.split()).split(",")]
        params = [] if params == ["void"] else params
        out[name] = (_letter(ret), "".join(_letter(p.rsplit(" ", 1)[0]) for p in params))
    return out


def test_signature_table_matches_the_headers():
    declared = {}
    for path in HEADERS:
        sigs = _header_signatures(path)
        assert not set(sigs) & set(declared), f"{path} declares {sorted(set(sigs) & set(declared))} again"
        declared.update(sigs)
        if path != MAIN_HEADER:
            assert '#include "metrics_b200.h"' in open(path).read(), path
    assert _native.SIGNATURES == declared


def test_library_exports_every_declared_symbol():
    assert os.path.exists(_native.lib_path()), "build the extension first: python -c 'import __graft_entry__ as g; g.build()'"
    raw = ctypes.CDLL(_native.lib_path())
    missing = [n for n in _native.SIGNATURES if not hasattr(raw, n)]
    assert not missing, f"symbols declared in the headers but not exported: {missing}"
    handle = _native.lib()
    for name, (ret, args) in _native.SIGNATURES.items():
        fn = getattr(handle, name)
        assert fn.restype is _native._C_TYPES[ret] and len(fn.argtypes) == len(args), name
    assert handle.mb200_abi_version() == _native.ABI_VERSION == 1
    assert isinstance(handle.mb200_last_error(), bytes)


def test_header_constants_match_the_binding():
    """Each Python mirror has the name of its header constant without the `MB200_` prefix."""
    text = "".join(_source(p) for p in HEADERS)
    found = re.findall(r"#define\s+MB200_(\w+)\s+(-?\d+)(?:u|ll)?\b", text) + re.findall(r"\bMB200_(\w+)\s*=\s*(-?\d+)", text)
    header = {name: int(value) for name, value in found}
    mirrors = ("ABI_VERSION F32 F16 BF16 F64 I64 I32 I16 I8 U8 BOOL FLAG_TARGET_RANGE FLAG_PREDS_RANGE FLAG_SPIN_TIMEOUT "
               "FLAG_CAPACITY SEG_PREDS_NEGATIVE SEG_PREDS_TOO_LARGE SEG_TARGET_NEGATIVE SEG_TARGET_TOO_LARGE RET_AP RET_RR "
               "RET_PRECISION RET_RECALL RET_HIT_RATE RET_FALL_OUT RET_R_PRECISION RET_NDCG RET_MAX_ELEMENTS RANKCORR_MAX_ROWS "
               "PQ_UNKNOWN_PREDS HD_PREDS_NOT_BINARY HD_TARGET_NOT_BINARY HD_NO_EDGES").split()
    assert {k: getattr(_native, k) for k in mirrors} == {k: header[k] for k in mirrors}
    assert _native.KENDALL_VARIANT == {v: header["KENDALL_" + v.upper()] for v in "abc"}
    assert _native.KENDALL_ALTERNATIVE == {a: header["KENDALL_ALT_" + (a or "none").upper().replace("-", "_")]
                                           for a in (None, "two-sided", "less", "greater")}
    # every other MB200_HD_* constant is a metric
    assert _native.HD_METRICS == {k[3:].lower(): v for k, v in header.items() if k.startswith("HD_") and k not in mirrors}


class _Recorder:
    """Stands in for the loaded library on a box without a GPU: every entry point of `_native.SIGNATURES` is a REAL ctypes
    function pointer with the declared signature around a Python callback, so a wrapper that passes the wrong
    number or kind of arguments fails here exactly as it would against the library.  Each call is recorded under the drive
    that made it, `calls[drive][name]`, and returns `answers[name](arguments)`: by default 256 for a size query and 0
    (success) for everything else."""

    def __init__(self, answers):
        self.calls = {}
        self.drive = None
        for name, (ret, args) in _native.SIGNATURES.items():
            sized = name.endswith(("_bytes", "_doubles", "_words"))

            def callback(*values, _name=name, _answer=answers.get(name, (lambda v: 256) if sized else (lambda v: 0))):
                self.calls.setdefault(self.drive, {}).setdefault(_name, []).append(values)
                return _answer(values)

            setattr(self, name, ctypes.CFUNCTYPE(_native._C_TYPES[ret], *[_native._C_TYPES[a] for a in args])(callback))


def _error_word(flags=0):
    """Answer of `mb200_panoptic_update`: like the library it overwrites its error word (argument 20), with `flags`, which
    the wrapper reads back."""
    def answer(values):
        ctypes.c_uint32.from_address(values[20]).value = flags
        return 0

    return answer


def _patch_host(monkeypatch, stream):
    """Host tensors stand in for device ones: the wrappers' device checks and stream query are patched out."""
    cpu = torch.device("cpu")
    monkeypatch.setattr(_native, "require_cuda", lambda *t: cpu)
    monkeypatch.setattr(_native, "on_device", lambda d: _native._NOOP)
    monkeypatch.setattr(_native, "stream_handle", lambda d: stream)
    monkeypatch.setattr(_native, "_flag_words", {})


def _panoptic_update(shape=(3, 5, 7, 2)):
    """K18 on zero maps: int64 preds, uint8 target, things {1, 3} and stuffs {2, 9}, modified PQ."""
    states = (torch.zeros(4, dtype=torch.float64), *(torch.zeros(4, dtype=torch.int32) for _ in range(3)))
    cats = _native.panoptic_categories({1, 3}, {2, 9}, torch.device("cpu"))
    return _native.panoptic_update_(*states, torch.zeros(shape, dtype=torch.int64), torch.zeros(shape, dtype=torch.uint8), cats,
                                    2, True, False)


N, C = 16, 3


def _drives():
    """{name: call} of every wrapper of `_native.py` and every `PeerWorkspace` method, on host tensors; each call is
    self-contained, so that it reaches the library on its own."""
    n, c = N, C
    scores, labels = torch.rand(n, c), torch.randint(c, (n,))
    i64 = lambda *shape: torch.zeros(*shape, dtype=torch.int64)  # noqa: E731
    i32 = lambda *shape: torch.zeros(*shape, dtype=torch.int32)  # noqa: E731
    # tp, fp, tn, fn and the workspace of the multiclass stat-score updates
    stats = lambda: (i64(c), i64(c), i64(c), i64(c), i64(3 * c + 2))  # noqa: E731
    flag = i32(1)
    boxes = torch.rand(4, 4)
    coco = (boxes, torch.rand(4), i64(4), [2, 2], boxes, i64(4), torch.zeros(4, dtype=torch.uint8), torch.ones(4), [2, 2], i64(1))
    # K10: the peer-memory exchange wrappers live on the workspace object (metrics_b200/peer.py); drive them on a bare one
    from metrics_b200 import peer

    ws = peer.PeerWorkspace.__new__(peer.PeerWorkspace)
    ws.device, ws.nbytes, ws.world, ws.rank, ws.table = torch.device("cpu"), 1 << 20, 2, 0, 0x1000
    masks = torch.rand(4, 5, 7) > 0.5
    off = torch.arange(4, dtype=torch.int64) * 2  # two 32-bit words per 5 x 7 mask
    img_off = torch.tensor([0, 2, 4], dtype=torch.int32)
    lab = torch.randint(0, 4, (3, 5, 6))
    oh = torch.nn.functional.one_hot(lab, 4).movedim(-1, 1)
    planar = oh.contiguous().bool()
    cl = oh.to(torch.uint8)
    strided = torch.rand(6, 4, 5, 6)[::2]
    groups = _native.RetrievalGroups(i64(n), torch.rand(n), i64(n + 1), i64(2), 1, 0)

    def hausdorff_one_hot():
        # a cap of four of the recorder's 1000-byte pairs, so that the 9 pairs do not fit one launch
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(_native, "HAUSDORFF_SCRATCH_BYTES", 4000)
            preds = torch.zeros(3, 4, 5, 7, dtype=torch.uint8).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
            return _native.hausdorff_distance(preds, torch.zeros(3, 4, 5, 7, dtype=torch.int32), 4, False, True, "taxicab",
                                              [2, 0.5], True)

    return {
        "confmat": lambda: _native.multiclass_confmat_update_(i64(c, c), scores, labels, c, 1, flag),
        "confmat_labels": lambda: _native.multiclass_confmat_update_(i64(c, c), labels, labels, c, None, None),
        "stat_scores": lambda: _native.multiclass_stat_scores_update_(*stats(), scores, labels, c, None, False, flag),
        "stat_scores_micro": lambda: _native.multiclass_stat_scores_update_(*stats(), scores, labels, c, None, True, None),
        "stats_softmax": lambda: _native.multiclass_stats_softmax_update_(*stats(), scores, labels, c, False, flag),
        "topk": lambda: _native.multiclass_stat_scores_topk_update_(*stats(), scores, labels, c, 2, None, None),
        "samplewise": lambda: _native.multiclass_stat_scores_samplewise(scores.reshape(4, c, 4), labels.reshape(4, 4), c, None, flag),
        "argmax": lambda: _native.argmax_rows(scores),
        "sigmoid": lambda: _native.sigmoid_if_logits(scores[:, 0]),
        "sigmoid_large": lambda: _native.sigmoid_if_logits(torch.rand(40000)),
        "softmax": lambda: _native.softmax_if_logits(scores),
        "softmax_f64": lambda: _native.softmax_if_logits(scores.double()),
        "curve": lambda: _native.curve_evaluate(scores[:, 0], labels.clamp(max=1), 1, 1, want_curve=True),
        "curve_ovr": lambda: _native.curve_evaluate(scores, labels, c, unit_range=False),
        "curve_ovr_unit_range": lambda: _native.curve_evaluate(scores, labels, c),
        "pack_keys": lambda: _native.curve_pack_keys(scores, c),
        "curve_keys": lambda: _native.curve_evaluate_keys(i32(c, n), labels, 0),
        "curve_keys_nonneg": lambda: _native.curve_evaluate_keys(i32(c, n), labels, 0, nonneg=True),
        "curve_multilabel": lambda: _native.curve_evaluate_multilabel(scores, torch.randint(2, (n, c)), c, ignore_index=-1, want_curve=True),
        "curve_multilabel_no_curve": lambda: _native.curve_evaluate_multilabel(scores, torch.randint(2, (n, c)), c, ignore_index=-1),
        "curve_weighted": lambda: _native.curve_weighted_clf_curve(scores[:, 0].double(), labels.clamp(max=1), torch.rand(n), 1),
        "binary_counts": lambda: _native.binary_stat_counts(scores, torch.randint(2, (n, c)), c, 0.5, None, False, None, flag),
        "binary_counts_samplewise": lambda: _native.binary_stat_counts(scores[:, 0], torch.randint(2, (n,)), 1, 0.5, 0, True),
        "regression": lambda: _native.regression_sums(scores[:, 0], scores[:, 1], _native.REG_MSE),
        "regression_columns": lambda: _native.regression_sums(scores, scores, _native.REG_R2, c),
        "tweedie": lambda: _native.regression_sums(scores[:, 0] + 0.1, scores[:, 1] + 0.1, _native.REG_TWEEDIE, 1, 1.5),
        "kl_divergence": lambda: _native.kl_divergence_rows(scores, scores + 1.0, False),  # K13
        "binned": lambda: _native.binned_curve_update(scores[:, 0], labels.clamp(max=1), torch.linspace(0, 1, 5), 1),
        "binned_multilabel": lambda: _native.binned_curve_update(scores, torch.randint(2, (n, c)), torch.linspace(0, 1, 5), c, multilabel=True),
        "peer_put_all": lambda: ws.put_all(labels, 256),
        "peer_pack_keys_put": lambda: ws.pack_keys_put(scores, 2, 2 * n, n, 0),
        "peer_reduce_put_i64": lambda: ws.reduce_put_i64(0, 4096, 100, 0),
        # K8 and K12: COCO mAP on boxes and instance masks
        "coco": lambda: _native.coco_map_evaluate(*coco, False, [0.5, 0.75], [0.0, 0.5, 1.0], [1, 10, 100]),
        "coco_match": lambda: _native.coco_map_match(*coco, [0.5, 0.75], 100),
        "coco_accumulate": lambda: _native.coco_map_accumulate(i32(4), torch.rand(4), i32(4), i64(4), i64(4), i32(1, 4), 1, 0, 1, 2,
                                                               [0.0, 0.5, 1.0], [1, 10, 100]),
        "mask_pack_bits": lambda: _native.mask_pack_bits(masks),
        "mask_pack_entry": lambda: _native.mask_pack_entry(masks),
        "mask_pair_intersections": lambda: _native.mask_pair_intersections(i32(8), off, i32(8), off, img_off, img_off,
                                                                           torch.tensor([2, 2], dtype=torch.int32), i64(4), i64(4),
                                                                           False, torch.tensor([0, 4]), 8, 4),
        "coco_match_masks": lambda: _native.coco_map_match(*coco, [0.5, 0.75], 100, micro=True, gt_area_exact=True, masks={
            "pair_inter": torch.zeros(8, dtype=torch.float64), "pair_off": torch.tensor([0, 4]),
            "det_area": torch.zeros(4, dtype=torch.float64), "gt_area": torch.zeros(4, dtype=torch.float64)}),
        # K14: calibration error
        "calibration_top_label": lambda: _native.calibration_top_label(scores, labels),
        "calibration_top_label_checked": lambda: _native.calibration_top_label(scores.double(), labels.int(), -1, flag),
        "calibration_top_label_ignore": lambda: _native.calibration_top_label(scores, labels, -1, flag),
        "calibration_top_label_wide": lambda: _native.calibration_top_label(torch.rand(4, 1500), labels[:4]),
        "calibration_top_label_f64": lambda: _native.calibration_top_label(scores.double(), labels),
        "calibration_bin_sums": lambda: _native.calibration_bin_sums(scores[:, 0], labels, torch.linspace(0, 1, 16)),
        "calibration_bin_sums_f16": lambda: _native.calibration_bin_sums(scores[:, 0].half(), labels.bool(), torch.linspace(0, 1, 101).half()),
        # K15: segmentation overlap counts
        "segmentation_index": lambda: _native.segmentation_overlap_counts(lab, lab, 4, True, True, True, flag),
        "segmentation_index_wide": lambda: _native.segmentation_overlap_counts(lab, lab, 5000, True, False, False),
        "segmentation_planar": lambda: _native.segmentation_overlap_counts(planar, planar, 9, False, False, False),
        "segmentation_channels_last": lambda: _native.segmentation_overlap_counts(cl, cl, 4, False, True, True),
        "segmentation_bool_channels_last": lambda: _native.segmentation_overlap_counts(oh.bool(), oh.bool(), 4, False, False, True),
        "segmentation_i64_planar": lambda: _native.segmentation_overlap_counts(oh.contiguous(), oh.contiguous(), 4, False, True, False),
        "segmentation_f16": lambda: _native.segmentation_overlap_counts(oh.half(), oh.half(), 4, False, True, False),
        "segmentation_strided": lambda: _native.segmentation_overlap_counts(strided, strided, 4, False, True, False),
        "segmentation_mixed": lambda: _native.segmentation_overlap_counts(cl, planar.to(torch.uint8), 4, False, True, False),
        # K16: retrieval (the device words read back are zeros on host tensors)
        "retrieval_sort": lambda: _native.retrieval_sort(torch.randint(3, (n,)), scores[:, 0], labels.clamp(max=1)),
        "retrieval_sort_one_query": lambda: _native.retrieval_sort(None, scores[:, 0], scores[:, 1]),
        "retrieval_sort_ideal": lambda: _native.retrieval_sort_ideal(groups),
        "retrieval_evaluate": lambda: _native.retrieval_evaluate(groups, _native.RET_NDCG, 3, True, torch.rand(n)),
        "retrieval_auroc": lambda: _native.retrieval_auroc(groups, None, 0.5),
        "retrieval_auroc_top_k": lambda: _native.retrieval_auroc(groups, 2, 0.5),
        "retrieval_pr_curve": lambda: _native.retrieval_pr_curve(groups, 4, adaptive_k=True),
        "retrieval_pr_curve_fixed_k": lambda: _native.retrieval_pr_curve(groups, 4),
        # K17: rank correlations
        "spearman": lambda: _native.spearman_corrcoef(scores[:, 0], scores[:, 1], torch.float64),
        "spearman_f32": lambda: _native.spearman_corrcoef(scores[:, 0], scores[:, 1], torch.float32),
        "kendall": lambda: _native.kendall_rank_corrcoef(scores, torch.randint(5, (n, c)), "b", "less"),
        "kendall_two_sided": lambda: _native.kendall_rank_corrcoef(scores, torch.randint(5, (n, c)), "b", "two-sided"),
        # K18: panoptic quality; K19: Hausdorff distance
        "panoptic": _panoptic_update,
        "hausdorff_one_hot": hausdorff_one_hot,
        "hausdorff_index": lambda: _native.hausdorff_distance(i64(2, 9, 6).transpose(1, 2), i64(2, 9, 6).transpose(1, 2), 5, True,
                                                              False, "euclidean", [1, 1], False),
    }


DRIVES = _drives()


def test_every_kernel_wrapper_calls_the_abi_as_declared(monkeypatch):
    """Run every drive once (CPU tensors, device checks patched out, library replaced by `_Recorder`): argument count and C
    types must match the headers, pointers must be non-NULL where a tensor was passed, and the stream handle must arrive as
    the last argument."""
    real = _native.lib()
    seg_sizes = {(fmt, dt): real.mb200_segmentation_scratch_bytes(4, 19, 4096, fmt, 1, dt, 0)
                 for fmt in (0, 1) for dt in (_native.F16, _native.BOOL)}
    assert seg_sizes[(1, _native.F16)] > 0 and seg_sizes[(0, _native.F16)] == seg_sizes[(1, _native.BOOL)] == 0
    fake = _Recorder({
        # like the library, the recorder asks for segmentation scratch only for float sums
        "mb200_segmentation_scratch_bytes": lambda v: 256 if v[5] == _native.F32 else 0,
        "mb200_panoptic_update": _error_word(),
        "mb200_hausdorff_scratch_bytes": lambda v: 1000 * v[3],
    })
    monkeypatch.setattr(_native, "lib", lambda: fake)
    _patch_host(monkeypatch, STREAM)
    results = {}
    for name, drive in DRIVES.items():
        fake.drive = name
        results[name] = drive()
    assert _native.launch_count() == 0

    # (`mb200_regression_num_sums` is a query for C callers; the Python mirror knows the layout of each op's sums)
    kernels = {k for k in _native.SIGNATURES if k not in ("mb200_abi_version", "mb200_last_error", "mb200_regression_num_sums",
                                                          "mb200_curve_workspace_bytes", "mb200_binary_stat_counts")}
    never_called = sorted(kernels - {name for calls in fake.calls.values() for name in calls})
    assert not never_called, f"no wrapper exercised: {never_called}"
    for drive, calls in fake.calls.items():
        for name, values_list in calls.items():
            args = _native.SIGNATURES[name][1]
            for values in values_list:
                assert len(values) == len(args), (drive, name)
                assert not args.endswith("p") or values[-1] == STREAM, f"{drive}: {name}: stream handle is not the last argument"
                assert not args.startswith("p") or values[0] not in (None, 0), f"{drive}: {name}: first pointer is NULL"

    def call(drive, name):
        (values,) = fake.calls[drive][name]
        return values

    # optional pointers really arrive as NULL, required ones as addresses
    with_flag, without_flag = call("confmat", "mb200_multiclass_confmat_update"), call("confmat_labels", "mb200_multiclass_confmat_update")
    assert with_flag[11] not in (None, 0) and without_flag[11] in (None, 0)
    assert with_flag[8] == 1 and with_flag[9] == 1 and without_flag[8] == 0
    counts_call = call("binary_counts", "mb200_binary_stat_counts_scratch")
    assert counts_call[7] == 0.5 and isinstance(counts_call[7], float)

    plain, checked = call("calibration_top_label", "mb200_calibration_top_label"), call("calibration_top_label_checked", "mb200_calibration_top_label")
    assert plain[1] == _native.F32 and checked[1] == _native.F64 and checked[3] == _native.I32
    assert (plain[4], plain[5]) == (16, 3)
    assert plain[6] == 0 and checked[6] == 1 and checked[7] == -1
    assert plain[12] in (None, 0) and checked[12] not in (None, 0)
    bins = call("calibration_bin_sums", "mb200_calibration_bin_sums")
    assert bins[4] == 16 and bins[6] == 15 and bins[1] == _native.F32 and bins[3] == _native.I64

    segmentation = [d for d in DRIVES if d.startswith("segmentation_")]
    for drive in segmentation:
        size, v = call(drive, "mb200_segmentation_scratch_bytes"), call(drive, "mb200_segmentation_overlap_counts")
        assert v[13] not in (None, 0)
        assert size[:5] == (v[4], v[5], v[6], v[7], v[8]) and size[5] == v[1] and size[6] == v[12]
    idx, pl, chl, st, mixed = (call("segmentation_" + d, "mb200_segmentation_overlap_counts")
                               for d in ("index", "planar", "channels_last", "strided", "mixed"))
    assert idx[1] == idx[3] == _native.I64 and idx[4:8] == (3, 4, 30, 0) and idx[9:13] == (30, 30, 1, 1)
    assert idx[16] not in (None, 0) and idx[14] in (None, 0) and idx[15] == 0
    assert pl[1] == _native.BOOL and pl[4:9] == (3, 4, 30, 1, 0) and pl[11:13] == (0, 0) and pl[16] in (None, 0)
    assert chl[1] == _native.U8 and chl[8] == 1 and chl[9:11] == (120, 120)
    assert st[1] == _native.F32 and st[8] == 0 and st[9] == 240  # a batch-strided planar view is read in place
    assert st[14] not in (None, 0) and st[15] == 256  # float sums get the scratch the library asked for
    assert mixed[8] == 0 and mixed[9:11] == (120, 120)

    by_index, one_query = call("retrieval_sort", "mb200_retrieval_sort"), call("retrieval_sort_one_query", "mb200_retrieval_sort")
    assert by_index[3] == _native.I64 and one_query[3] == _native.F32 and by_index[4] == one_query[4] == N
    evaluate = call("retrieval_evaluate", "mb200_retrieval_evaluate")
    assert evaluate[2] not in (None, 0) and evaluate[5:9] == (N, _native.RET_NDCG, 3, 1) and evaluate[12] == 256
    auroc = call("retrieval_auroc", "mb200_retrieval_auroc")
    assert auroc[4:7] == (N, 0, 0.5) and auroc[10] == 256
    curve = call("retrieval_pr_curve", "mb200_retrieval_pr_curve")
    assert curve[4:7] == (N, 4, 1) and curve[11] == 256

    spearman = call("spearman", "mb200_spearman_corrcoef")
    assert (spearman[1], spearman[3], spearman[4:6], spearman[7], spearman[8]) == (_native.F32, _native.F32, (N, 1), _native.F64, 1e-6)
    kendall = call("kendall", "mb200_kendall_rank_corrcoef")
    assert (kendall[1], kendall[3], kendall[4:8], kendall[9]) == (_native.F32, _native.I64, (N, C, 1, 2), _native.F32)
    assert kendall[10] not in (None, 0)

    assert results["panoptic"] is False
    pq = call("panoptic", "mb200_panoptic_update")
    assert pq[1] == _native.I64 and pq[3] == _native.U8 and pq[4:6] == (3, 35)
    assert pq[7:11] == (4, 2, 1, 0)  # categories, things, modified, allow_unknown_preds
    assert pq[11:14] == (3, 128, 128)  # all images in one launch; tables no larger than 2 * pixels needs
    assert all(v not in (None, 0) for v in (pq[0], pq[2], pq[6], *pq[14:19], pq[20]))

    out, err = results["hausdorff_one_hot"]
    assert out.shape == (3, 3) and out.dtype == torch.float32 and err.shape == (2,) and err.dtype == torch.int64
    hd = call("hausdorff_one_hot", "mb200_hausdorff_distance")
    assert hd[1] == _native.U8 and hd[3] == _native.I32 and hd[4:9] == (1, 3, 4, 5, 7)
    assert hd[9:13] == (140, 1, 28, 4) and hd[13:17] == (140, 35, 7, 1)  # channels-last preds, contiguous target
    assert hd[17:23] == (1, 2, 1, 2.0, 0.5, 1)  # drop background, taxicab, axis 0 int, spacing, directed
    assert hd[23] == 4 and hd[26] == 4000  # pairs per launch under the scratch cap, the scratch of that launch
    assert all(v not in (None, 0) for v in (hd[0], hd[2], hd[24], hd[25], hd[27]))
    index = call("hausdorff_index", "mb200_hausdorff_distance")  # index labels pass three strides
    assert index[4:9] == (0, 2, 5, 6, 9) and index[9:13] == (54, 0, 1, 6) and index[19] == 3 and index[23] == 10


def test_real_library_accepts_every_wrappers_arguments_up_to_the_first_cuda_call(monkeypatch):
    """GPU-less boxes only.  Every drive is run against the REAL `.so` with host tensors (device checks patched out):
    ctypes conversion, the library's own argument validation (`MB200_REQUIRE`) and its host-side set-up must all pass, so the
    first failure has to be a CUDA runtime error (code -2, no driver) — never an argument error (-1 / ValueError / TypeError)."""
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present: host pointers must not reach the kernels")
    _patch_host(monkeypatch, 0)
    for name, drive in DRIVES.items():
        with pytest.raises(_native.NativeLibraryError, match=r"\(code -2\): CUDA error"):
            drive()


def test_library_rejects_bad_calibration_arguments(monkeypatch):
    """Argument errors are ValueErrors raised before any CUDA call (works with and without a device: host tensors)."""
    _patch_host(monkeypatch, 0)
    with pytest.raises(ValueError, match="n_bins must lie in"):
        _native.calibration_bin_sums(torch.rand(4), torch.ones(4), torch.linspace(0, 1, 9000))
    with pytest.raises(ValueError, match="preds must be"):
        _native.calibration_top_label(torch.randint(3, (4, 3)), torch.zeros(4, dtype=torch.long))
    with pytest.raises(ValueError, match="target must be an integer"):
        _native.calibration_top_label(torch.rand(4, 3), torch.zeros(4))


def test_library_rejects_bad_segmentation_arguments(monkeypatch):
    _patch_host(monkeypatch, 0)
    lab = torch.randint(0, 4, (3, 5))
    with pytest.raises(ValueError, match="index labels must be int64"):
        _native.segmentation_overlap_counts(lab.int(), lab.int(), 4, True, True, True)
    with pytest.raises(ValueError, match="only the product"):
        _native.segmentation_overlap_counts(torch.rand(2, 3, 4), torch.rand(2, 3, 4), 3, False, False, True)
    with pytest.raises(ValueError, match="unsupported dtype"):
        _native.segmentation_overlap_counts(torch.rand(2, 3, 4).double(), torch.rand(2, 3, 4).double(), 3, False, True, True)
