"""CPU: the segmentation C-ABI (include/metrics_b200_segmentation.h) and its ctypes table `_native.SEGMENTATION_SIGNATURES`,
checked the way tests/test_calibration_abi.py checks the calibration header."""
import ctypes
import os
import re

import pytest
import torch

from tests.conftest import ROOT
from tests.test_calibration_abi import _letter, _patch_host

HEADER = os.path.join(ROOT, "include", "metrics_b200_segmentation.h")


def _header_signatures():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    out = {}
    for ret, name, args in re.findall(r"MB200_API\s+([\w\s\*]+?)\s*(mb200_\w+)\s*\(([^)]*)\)\s*;", text):
        params = [a.strip() for a in " ".join(args.split()).split(",")]
        out[name] = (_letter(ret), "".join(_letter(p.rsplit(" ", 1)[0]) for p in params))
    return out


def _header_defines():
    return {k: int(v.rstrip("u")) for k, v in re.findall(r"#define (MB200_SEG_\w+) (\d+u?)", open(HEADER).read())}


def test_table_matches_the_header_and_the_library_exports_it():
    from metrics_b200 import _native

    assert '#include "metrics_b200.h"' in open(HEADER).read()
    assert _native.SEGMENTATION_SIGNATURES == _header_signatures()
    main = open(os.path.join(ROOT, "include", "metrics_b200.h")).read()
    assert not set(_header_signatures()) & set(re.findall(r"MB200_API[^;(]*?\b(mb200_\w+)\s*\(", main))
    raw = ctypes.CDLL(_native.lib_path())
    assert all(hasattr(raw, n) for n in _native.SEGMENTATION_SIGNATURES)
    for name, (ret, args) in _native.SEGMENTATION_SIGNATURES.items():
        fn = getattr(_native.lib(), name)
        assert fn.restype is _native._C_TYPES[ret] and len(fn.argtypes) == len(args), name
    d = _header_defines()
    sizes = {(fmt, dt): _native.lib().mb200_segmentation_scratch_bytes(4, 19, 4096, fmt, 1, dt, 0)
             for fmt in (0, 1) for dt in (_native.F16, _native.BOOL)}
    assert sizes[(1, _native.F16)] > 0 and sizes[(0, _native.F16)] == sizes[(1, _native.BOOL)] == 0
    assert (d["MB200_SEG_PREDS_NEGATIVE"], d["MB200_SEG_PREDS_TOO_LARGE"], d["MB200_SEG_TARGET_NEGATIVE"],
            d["MB200_SEG_TARGET_TOO_LARGE"]) == (_native.SEG_PREDS_NEGATIVE, _native.SEG_PREDS_TOO_LARGE,
                                                 _native.SEG_TARGET_NEGATIVE, _native.SEG_TARGET_TOO_LARGE)


class _Recorder:
    """Both entry points as real ctypes function pointers with the declared signatures around a recorder."""

    def __init__(self, native):
        self.calls, self._keep = {}, []
        for name, (ret, args) in native.SEGMENTATION_SIGNATURES.items():
            proto = ctypes.CFUNCTYPE(native._C_TYPES[ret], *[native._C_TYPES[a] for a in args])

            def callback(*values, _name=name):
                self.calls.setdefault(_name, []).append(values)
                return (256 if values[5] == native.F32 else 0) if _name.endswith("_bytes") else 0

            fn = proto(callback)
            self._keep.append(fn)
            setattr(self, name, fn)


def test_wrapper_calls_the_abi_as_declared(monkeypatch):
    from metrics_b200 import _native

    fake = _Recorder(_native)
    monkeypatch.setattr(_native, "lib", lambda: fake)
    _patch_host(monkeypatch, _native, 0xBEEF)
    lab = torch.randint(0, 4, (3, 5, 6))
    flag = torch.zeros(1, dtype=torch.int32)
    planar = torch.nn.functional.one_hot(lab, 4).movedim(-1, 1).contiguous().bool()
    cl = torch.nn.functional.one_hot(lab, 4).movedim(-1, 1).to(torch.uint8)
    strided = torch.rand(6, 4, 5, 6)[::2]
    _native.segmentation_overlap_counts(lab, lab, 4, True, True, True, flag)
    _native.segmentation_overlap_counts(planar, planar, 9, False, False, False)
    _native.segmentation_overlap_counts(cl, cl, 4, False, True, True)
    _native.segmentation_overlap_counts(strided, strided, 4, False, True, False)
    _native.segmentation_overlap_counts(cl, planar.to(torch.uint8), 4, False, True, False)  # mixed layouts: one copy each
    assert set(fake.calls) == set(_native.SEGMENTATION_SIGNATURES)
    sizes, calls = fake.calls["mb200_segmentation_scratch_bytes"], fake.calls["mb200_segmentation_overlap_counts"]
    assert len(calls) == 5 and len(sizes) == 5
    for v in calls:
        assert len(v) == 18 and v[-1] == 0xBEEF and v[0] not in (None, 0) and v[13] not in (None, 0)
    for size, v in zip(sizes, calls):
        assert size[:5] == (v[4], v[5], v[6], v[7], v[8]) and size[5] == v[1] and size[6] == v[12]
    idx, pl, chl, st, mixed = calls
    assert idx[1] == idx[3] == _native.I64 and idx[4:8] == (3, 4, 30, 0) and idx[9:13] == (30, 30, 1, 1)
    assert idx[16] not in (None, 0) and idx[14] in (None, 0) and idx[15] == 0
    assert pl[1] == _native.BOOL and pl[4:9] == (3, 4, 30, 1, 0) and pl[11:13] == (0, 0) and pl[16] in (None, 0)
    assert chl[1] == _native.U8 and chl[8] == 1 and chl[9:11] == (120, 120)
    assert st[1] == _native.F32 and st[8] == 0 and st[9] == 240  # a batch-strided planar view is read in place
    assert st[14] not in (None, 0) and st[15] == 256  # float sums get the scratch the library asked for
    assert mixed[8] == 0 and mixed[9:11] == (120, 120)


def test_real_library_accepts_the_arguments_up_to_the_first_cuda_call(monkeypatch):
    """GPU-less boxes only: argument conversion and the library's own checks pass, the first failure is a CUDA error."""
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present: host pointers must not reach the kernels")
    from metrics_b200 import _native

    _patch_host(monkeypatch, _native, 0)
    lab = torch.randint(0, 4, (3, 5, 6))
    oh = torch.nn.functional.one_hot(lab, 4).movedim(-1, 1)
    calls = {
        "index": lambda: _native.segmentation_overlap_counts(lab, lab, 4, True, True, True, torch.zeros(1, dtype=torch.int32)),
        "index_wide": lambda: _native.segmentation_overlap_counts(lab, lab, 5000, True, False, False),
        "bool_cl": lambda: _native.segmentation_overlap_counts(oh.bool(), oh.bool(), 4, False, False, True),
        "i64_planar": lambda: _native.segmentation_overlap_counts(oh.contiguous(), oh.contiguous(), 4, False, True, False),
        "f16": lambda: _native.segmentation_overlap_counts(oh.half(), oh.half(), 4, False, True, False),
    }
    for name, call in calls.items():
        with pytest.raises(_native.NativeLibraryError, match=r"\(code -2\): CUDA error"):
            call()


def test_library_rejects_bad_arguments(monkeypatch):
    from metrics_b200 import _native

    _patch_host(monkeypatch, _native, 0)
    lab = torch.randint(0, 4, (3, 5))
    with pytest.raises(ValueError, match="index labels must be int64"):
        _native.segmentation_overlap_counts(lab.int(), lab.int(), 4, True, True, True)
    with pytest.raises(ValueError, match="only the product"):
        _native.segmentation_overlap_counts(torch.rand(2, 3, 4), torch.rand(2, 3, 4), 3, False, False, True)
    with pytest.raises(ValueError, match="unsupported dtype"):
        _native.segmentation_overlap_counts(torch.rand(2, 3, 4).double(), torch.rand(2, 3, 4).double(), 3, False, True, True)
