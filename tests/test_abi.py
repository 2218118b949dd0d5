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
               "SEG_PREDS_NEGATIVE SEG_PREDS_TOO_LARGE SEG_TARGET_NEGATIVE SEG_TARGET_TOO_LARGE RET_AP RET_RR RET_PRECISION "
               "RET_RECALL RET_HIT_RATE RET_FALL_OUT RET_R_PRECISION RET_NDCG RET_MAX_ELEMENTS RANKCORR_MAX_ROWS").split()
    assert {k: getattr(_native, k) for k in mirrors} == {k: header[k] for k in mirrors}
    assert _native.KENDALL_VARIANT == {v: header["KENDALL_" + v.upper()] for v in "abc"}
    assert _native.KENDALL_ALTERNATIVE == {a: header["KENDALL_ALT_" + (a or "none").upper().replace("-", "_")]
                                           for a in (None, "two-sided", "less", "greater")}


class _Recorder:
    """Stands in for the loaded library on a box without a GPU: every entry point of `_native.SIGNATURES` is a REAL ctypes
    function pointer with the declared signature around a Python callback, so a wrapper that passes the wrong
    number or kind of arguments fails here exactly as it would against the library.  Each call is recorded and reports
    success; a size query answers `sizes[name](arguments)`, 256 when `sizes` has no entry for it."""

    def __init__(self, sizes):
        self.calls = {}
        for name, (ret, args) in _native.SIGNATURES.items():
            def callback(*values, _name=name):
                self.calls.setdefault(_name, []).append(values)
                if _name.endswith(("_bytes", "_doubles", "_words")):
                    return sizes.get(_name, lambda v: 256)(values)
                return 0

            setattr(self, name, ctypes.CFUNCTYPE(_native._C_TYPES[ret], *[_native._C_TYPES[a] for a in args])(callback))


def _patch_host(monkeypatch, stream):
    """Host tensors stand in for device ones: the wrappers' device checks and stream query are patched out."""
    cpu = torch.device("cpu")
    monkeypatch.setattr(_native, "require_cuda", lambda *t: cpu)
    monkeypatch.setattr(_native, "on_device", lambda d: _native._NOOP)
    monkeypatch.setattr(_native, "stream_handle", lambda d: stream)
    monkeypatch.setattr(_native, "_flag_words", {})


def test_every_kernel_wrapper_calls_the_abi_as_declared(monkeypatch):
    """Drive each wrapper of `_native.py` and each `PeerWorkspace` method once (CPU tensors, device checks patched out,
    library replaced by `_Recorder`): argument count and C types must match the headers, pointers must be non-NULL where a
    tensor was passed, and the stream handle must arrive as the last argument."""
    real = _native.lib()
    seg_sizes = {(fmt, dt): real.mb200_segmentation_scratch_bytes(4, 19, 4096, fmt, 1, dt, 0)
                 for fmt in (0, 1) for dt in (_native.F16, _native.BOOL)}
    assert seg_sizes[(1, _native.F16)] > 0 and seg_sizes[(0, _native.F16)] == seg_sizes[(1, _native.BOOL)] == 0
    # like the library, the recorder asks for segmentation scratch only for float sums
    fake = _Recorder({"mb200_segmentation_scratch_bytes": lambda v: 256 if v[5] == _native.F32 else 0})
    monkeypatch.setattr(_native, "lib", lambda: fake)
    _patch_host(monkeypatch, STREAM)

    n, c = 16, 3
    scores, labels = torch.rand(n, c), torch.randint(c, (n,))
    i64 = lambda *shape: torch.zeros(*shape, dtype=torch.int64)  # noqa: E731
    flag = torch.zeros(1, dtype=torch.int32)
    _native.multiclass_confmat_update_(i64(c, c), scores, labels, c, 1, flag)
    _native.multiclass_confmat_update_(i64(c, c), labels, labels, c, None, None)
    _native.multiclass_stat_scores_update_(i64(c), i64(c), i64(c), i64(c), i64(3 * c + 2), scores, labels, c, None, False, flag)
    _native.multiclass_stats_softmax_update_(i64(c), i64(c), i64(c), i64(c), i64(3 * c + 2), scores, labels, c, False, flag)
    _native.multiclass_stat_scores_topk_update_(i64(c), i64(c), i64(c), i64(c), i64(3 * c + 2), scores, labels, c, 2, None, None)
    _native.multiclass_stat_scores_samplewise(scores.reshape(4, c, 4), labels.reshape(4, 4), c, None, flag)
    _native.argmax_rows(scores)
    _native.sigmoid_if_logits(scores[:, 0])
    _native.sigmoid_if_logits(torch.rand(40000))
    _native.softmax_if_logits(scores)
    _native.softmax_if_logits(scores.double())
    _native.curve_evaluate(scores[:, 0], labels.clamp(max=1), 1, 1, want_curve=True)
    _native.curve_evaluate(scores, labels, c, unit_range=False)
    keys = _native.curve_pack_keys(scores, c)
    _native.curve_evaluate_keys(keys, labels, 0)
    _native.curve_evaluate_keys(keys, labels, 0, nonneg=True)
    _native.curve_evaluate_multilabel(scores, torch.randint(2, (n, c)), c, ignore_index=-1, want_curve=True)
    _native.binary_stat_counts(scores, torch.randint(2, (n, c)), c, 0.5, None, False, None, flag)
    _native.binary_stat_counts(scores[:, 0], torch.randint(2, (n,)), 1, 0.5, 0, True)
    _native.regression_sums(scores[:, 0], scores[:, 1], 0)
    _native.binned_curve_update(scores[:, 0], labels.clamp(max=1), torch.linspace(0, 1, 5), 1)
    _native.binned_curve_update(scores, torch.randint(2, (n, c)), torch.linspace(0, 1, 5), c, multilabel=True)
    boxes = torch.rand(4, 4)
    _native.coco_map_evaluate(boxes, torch.rand(4), torch.zeros(4, dtype=torch.long), [2, 2], boxes, torch.zeros(4, dtype=torch.long),
                              torch.zeros(4, dtype=torch.uint8), torch.ones(4), [2, 2], torch.zeros(1, dtype=torch.long), False,
                              [0.5, 0.75], [0.0, 0.5, 1.0], [1, 10, 100])
    _native.curve_weighted_clf_curve(scores[:, 0].double(), labels.clamp(max=1), torch.rand(n), 1)
    # K10: the peer-memory exchange wrappers live on the workspace object (metrics_b200/peer.py); drive them on a bare one
    from metrics_b200 import peer

    ws = peer.PeerWorkspace.__new__(peer.PeerWorkspace)
    ws.device, ws.nbytes, ws.world, ws.rank, ws.table = torch.device("cpu"), 1 << 20, 2, 0, 0x1000
    ws.put_all(labels, 256)
    ws.pack_keys_put(scores, 2, 2 * n, n, 0)
    ws.reduce_put_i64(0, 4096, 100, 0)
    recs, npig, _ = _native.coco_map_match(boxes, torch.rand(4), torch.zeros(4, dtype=torch.long), [2, 2], boxes,
                                           torch.zeros(4, dtype=torch.long), torch.zeros(4, dtype=torch.uint8), torch.ones(4), [2, 2],
                                           torch.zeros(1, dtype=torch.long), [0.5, 0.75], 100)
    _native.coco_map_accumulate(recs[0], torch.rand(4), recs[1], recs[2], recs[3], npig, 1, 0, 1, 2, [0.0, 0.5, 1.0], [1, 10, 100])
    _native.kl_divergence_rows(scores, scores + 1.0, False)  # K13
    # K12: instance masks
    words, area = _native.mask_pack_bits(torch.rand(4, 5, 7) > 0.5)
    _native.mask_pack_entry(torch.rand(4, 5, 7) > 0.5)
    off = torch.arange(4, dtype=torch.int64) * words.shape[1]
    img_off = torch.tensor([0, 2, 4], dtype=torch.int32)
    inter = _native.mask_pair_intersections(words.reshape(-1), off, words.reshape(-1), off, img_off, img_off,
                                            torch.tensor([2, 2], dtype=torch.int32), torch.zeros(4, dtype=torch.long),
                                            torch.zeros(4, dtype=torch.long), False, torch.tensor([0, 4]), 8, 4)
    _native.coco_map_match(boxes, torch.rand(4), torch.zeros(4, dtype=torch.long), [2, 2], boxes, torch.zeros(4, dtype=torch.long),
                           torch.zeros(4, dtype=torch.uint8), torch.ones(4), [2, 2], torch.zeros(1, dtype=torch.long), [0.5, 0.75], 100,
                           micro=True, masks={"pair_inter": inter, "pair_off": torch.tensor([0, 4]), "det_area": area.double(),
                                              "gt_area": area.double()}, gt_area_exact=True)
    # K14: calibration error
    _native.calibration_top_label(scores, labels)
    _native.calibration_top_label(scores.double(), labels.int(), -1, flag)
    _native.calibration_bin_sums(scores[:, 0], labels, torch.linspace(0, 1, 16))
    # K15: segmentation overlap counts
    lab = torch.randint(0, 4, (3, 5, 6))
    planar = torch.nn.functional.one_hot(lab, 4).movedim(-1, 1).contiguous().bool()
    cl = torch.nn.functional.one_hot(lab, 4).movedim(-1, 1).to(torch.uint8)
    strided = torch.rand(6, 4, 5, 6)[::2]
    _native.segmentation_overlap_counts(lab, lab, 4, True, True, True, flag)
    _native.segmentation_overlap_counts(planar, planar, 9, False, False, False)
    _native.segmentation_overlap_counts(cl, cl, 4, False, True, True)
    _native.segmentation_overlap_counts(strided, strided, 4, False, True, False)
    _native.segmentation_overlap_counts(cl, planar.to(torch.uint8), 4, False, True, False)  # mixed layouts: one copy each
    # K16: retrieval (the device words read back are zeros on host tensors)
    groups = _native.retrieval_sort(torch.randint(3, (n,)), scores[:, 0], labels.clamp(max=1))
    _native.retrieval_sort(None, scores[:, 0], scores[:, 1])
    ideal = _native.retrieval_sort_ideal(groups)
    _native.retrieval_evaluate(groups, _native.RET_NDCG, 3, True, ideal)
    _native.retrieval_auroc(groups, None, 0.5)
    _native.retrieval_pr_curve(groups, 4, adaptive_k=True)
    # K17: rank correlations
    _native.spearman_corrcoef(scores[:, 0], scores[:, 1], torch.float64)
    _native.kendall_rank_corrcoef(scores, torch.randint(5, (n, c)), "b", "less")
    assert _native.launch_count() == 0

    # (`mb200_regression_num_sums` is a query for C callers; the Python mirror knows the layout of each op's sums)
    kernels = {k for k in _native.SIGNATURES if k not in ("mb200_abi_version", "mb200_last_error", "mb200_regression_num_sums",
                                                          "mb200_curve_workspace_bytes", "mb200_binary_stat_counts")}
    never_called = sorted(kernels - set(fake.calls))
    assert not never_called, f"no wrapper exercised: {never_called}"
    for name, calls in fake.calls.items():
        args = _native.SIGNATURES[name][1]
        for values in calls:
            assert len(values) == len(args), name
            assert not args.endswith("p") or values[-1] == STREAM, f"{name}: stream handle is not the last argument"
            assert not args.startswith("p") or values[0] not in (None, 0), f"{name}: first pointer is NULL"
    # optional pointers really arrive as NULL, required ones as addresses
    with_flag, without_flag = fake.calls["mb200_multiclass_confmat_update"]
    assert with_flag[11] not in (None, 0) and without_flag[11] in (None, 0)
    assert with_flag[8] == 1 and with_flag[9] == 1 and without_flag[8] == 0
    counts_call = fake.calls["mb200_binary_stat_counts_scratch"][0]
    assert counts_call[7] == 0.5 and isinstance(counts_call[7], float)

    plain, checked = fake.calls["mb200_calibration_top_label"]
    assert plain[1] == _native.F32 and checked[1] == _native.F64 and checked[3] == _native.I32
    assert (plain[4], plain[5]) == (16, 3)
    assert plain[6] == 0 and checked[6] == 1 and checked[7] == -1
    assert plain[12] in (None, 0) and checked[12] not in (None, 0)
    bins = fake.calls["mb200_calibration_bin_sums"][0]
    assert bins[4] == 16 and bins[6] == 15 and bins[1] == _native.F32 and bins[3] == _native.I64

    sizes, calls = fake.calls["mb200_segmentation_scratch_bytes"], fake.calls["mb200_segmentation_overlap_counts"]
    assert len(calls) == 5 and len(sizes) == 5
    for size, v in zip(sizes, calls):
        assert v[13] not in (None, 0)
        assert size[:5] == (v[4], v[5], v[6], v[7], v[8]) and size[5] == v[1] and size[6] == v[12]
    idx, pl, chl, st, mixed = calls
    assert idx[1] == idx[3] == _native.I64 and idx[4:8] == (3, 4, 30, 0) and idx[9:13] == (30, 30, 1, 1)
    assert idx[16] not in (None, 0) and idx[14] in (None, 0) and idx[15] == 0
    assert pl[1] == _native.BOOL and pl[4:9] == (3, 4, 30, 1, 0) and pl[11:13] == (0, 0) and pl[16] in (None, 0)
    assert chl[1] == _native.U8 and chl[8] == 1 and chl[9:11] == (120, 120)
    assert st[1] == _native.F32 and st[8] == 0 and st[9] == 240  # a batch-strided planar view is read in place
    assert st[14] not in (None, 0) and st[15] == 256  # float sums get the scratch the library asked for
    assert mixed[8] == 0 and mixed[9:11] == (120, 120)

    by_index, one_query = fake.calls["mb200_retrieval_sort"]
    assert by_index[3] == _native.I64 and one_query[3] == _native.F32 and by_index[4] == one_query[4] == n
    evaluate = fake.calls["mb200_retrieval_evaluate"][0]
    assert evaluate[2] not in (None, 0) and evaluate[5:9] == (n, _native.RET_NDCG, 3, 1) and evaluate[12] == 256
    auroc = fake.calls["mb200_retrieval_auroc"][0]
    assert auroc[4:7] == (n, 0, 0.5) and auroc[10] == 256
    curve = fake.calls["mb200_retrieval_pr_curve"][0]
    assert curve[4:7] == (n, 4, 1) and curve[11] == 256

    spearman = fake.calls["mb200_spearman_corrcoef"][0]
    assert (spearman[1], spearman[3], spearman[4:6], spearman[7], spearman[8]) == (_native.F32, _native.F32, (n, 1), _native.F64, 1e-6)
    kendall = fake.calls["mb200_kendall_rank_corrcoef"][0]
    assert (kendall[1], kendall[3], kendall[4:8], kendall[9]) == (_native.F32, _native.I64, (n, c, 1, 2), _native.F32)
    assert kendall[10] not in (None, 0)


def test_real_library_accepts_every_wrappers_arguments_up_to_the_first_cuda_call(monkeypatch):
    """GPU-less boxes only.  Each wrapper is called against the REAL `.so` with host tensors (device checks patched out):
    ctypes conversion, the library's own argument validation (`MB200_REQUIRE`) and its host-side set-up must all pass, so the
    first failure has to be a CUDA runtime error (code -2, no driver) — never an argument error (-1 / ValueError / TypeError)."""
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present: host pointers must not reach the kernels")
    _patch_host(monkeypatch, 0)
    n, c = 16, 3
    scores, labels = torch.rand(n, c), torch.randint(c, (n,))
    i64 = lambda *shape: torch.zeros(*shape, dtype=torch.int64)  # noqa: E731
    flag = torch.zeros(1, dtype=torch.int32)
    boxes = torch.rand(4, 4)
    lab = torch.randint(0, 4, (3, 5, 6))
    oh = torch.nn.functional.one_hot(lab, 4).movedim(-1, 1)
    groups = _native.RetrievalGroups(i64(n), torch.rand(n), i64(n + 1), i64(2), 1, 0)
    calls = {
        "confmat": lambda: _native.multiclass_confmat_update_(i64(c, c), scores, labels, c, 1, flag),
        "stat_scores": lambda: _native.multiclass_stat_scores_update_(i64(c), i64(c), i64(c), i64(c), i64(3 * c + 2), scores, labels, c, None, True, None),
        "topk": lambda: _native.multiclass_stat_scores_topk_update_(i64(c), i64(c), i64(c), i64(c), i64(3 * c + 2), scores, labels, c, 2, None, None),
        "samplewise": lambda: _native.multiclass_stat_scores_samplewise(scores.reshape(4, c, 4), labels.reshape(4, 4), c, None, flag),
        "argmax": lambda: _native.argmax_rows(scores),
        "sigmoid": lambda: _native.sigmoid_if_logits(scores[:, 0]),
        "softmax": lambda: _native.softmax_if_logits(scores),
        "curve": lambda: _native.curve_evaluate(scores[:, 0], labels.clamp(max=1), 1, 1, want_curve=True),
        "curve_ovr": lambda: _native.curve_evaluate(scores, labels, c),
        "pack_keys": lambda: _native.curve_pack_keys(scores, c),
        "curve_multilabel": lambda: _native.curve_evaluate_multilabel(scores, torch.randint(2, (n, c)), c, ignore_index=-1),
        "binary_counts": lambda: _native.binary_stat_counts(scores, torch.randint(2, (n, c)), c, 0.5, None, False, None, flag),
        "regression": lambda: _native.regression_sums(scores[:, 0], scores[:, 1], _native.REG_MSE),
        "regression_columns": lambda: _native.regression_sums(scores, scores, _native.REG_R2, c),
        "tweedie": lambda: _native.regression_sums(scores[:, 0] + 0.1, scores[:, 1] + 0.1, _native.REG_TWEEDIE, 1, 1.5),
        "binned": lambda: _native.binned_curve_update(scores[:, 0], labels.clamp(max=1), torch.linspace(0, 1, 5), 1),
        "binned_multilabel": lambda: _native.binned_curve_update(scores, torch.randint(2, (n, c)), torch.linspace(0, 1, 5), c, multilabel=True),
        "coco": lambda: _native.coco_map_evaluate(boxes, torch.rand(4), torch.zeros(4, dtype=torch.long), [2, 2], boxes,
                                                  torch.zeros(4, dtype=torch.long), torch.zeros(4, dtype=torch.uint8), torch.ones(4), [2, 2],
                                                  torch.zeros(1, dtype=torch.long), False, [0.5, 0.75], [0.0, 0.5, 1.0], [1, 10, 100]),
        "calibration_top_label": lambda: _native.calibration_top_label(scores, labels, -1, flag),
        "calibration_top_label_wide": lambda: _native.calibration_top_label(torch.rand(4, 1500), labels[:4]),
        "calibration_top_label_f64": lambda: _native.calibration_top_label(scores.double(), labels),
        "calibration_bin_sums": lambda: _native.calibration_bin_sums(scores[:, 0], labels, torch.linspace(0, 1, 16)),
        "calibration_bin_sums_f16": lambda: _native.calibration_bin_sums(scores[:, 0].half(), labels.bool(), torch.linspace(0, 1, 101).half()),
        "segmentation_index": lambda: _native.segmentation_overlap_counts(lab, lab, 4, True, True, True, flag),
        "segmentation_index_wide": lambda: _native.segmentation_overlap_counts(lab, lab, 5000, True, False, False),
        "segmentation_bool_cl": lambda: _native.segmentation_overlap_counts(oh.bool(), oh.bool(), 4, False, False, True),
        "segmentation_i64_planar": lambda: _native.segmentation_overlap_counts(oh.contiguous(), oh.contiguous(), 4, False, True, False),
        "segmentation_f16": lambda: _native.segmentation_overlap_counts(oh.half(), oh.half(), 4, False, True, False),
        "retrieval_sort": lambda: _native.retrieval_sort(torch.randint(3, (n,)), scores[:, 0], labels.clamp(max=1)),
        "retrieval_sort_one_query": lambda: _native.retrieval_sort(None, scores[:, 0], scores[:, 1]),
        "retrieval_sort_ideal": lambda: _native.retrieval_sort_ideal(groups),
        "retrieval_evaluate": lambda: _native.retrieval_evaluate(groups, _native.RET_NDCG, 3, True, torch.rand(n)),
        "retrieval_auroc": lambda: _native.retrieval_auroc(groups, 2, 0.5),
        "retrieval_pr_curve": lambda: _native.retrieval_pr_curve(groups, 4),
        "spearman": lambda: _native.spearman_corrcoef(scores[:, 0], scores[:, 1], torch.float32),
        "kendall": lambda: _native.kendall_rank_corrcoef(scores, torch.randint(5, (n, c)), "b", "two-sided"),
    }
    for name, call in calls.items():
        with pytest.raises(_native.NativeLibraryError, match=r"\(code -2\): CUDA error"):
            call()


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
