"""CPU: the calibration-error C-ABI (include/metrics_b200_calibration.h) and its ctypes table
`_native.CALIBRATION_SIGNATURES` — the checks tests/test_native_abi.py gives the main header, for the companion one."""
import ctypes
import os
import re

import pytest
import torch

from tests.conftest import ROOT

HEADER = os.path.join(ROOT, "include", "metrics_b200_calibration.h")


def _letter(ctype: str) -> str:
    ctype = ctype.strip()
    if "char" in ctype and "*" in ctype:
        return "s"
    if "*" in ctype:
        return "p"
    return {"int": "i", "int64_t": "q", "uint64_t": "Q", "double": "d"}[ctype.replace("const", "").split()[0]]


def _header_signatures():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"//[^\n]*", "", text)
    out = {}
    for ret, name, args in re.findall(r"MB200_API\s+([\w\s\*]+?)\s*(mb200_\w+)\s*\(([^)]*)\)\s*;", text):
        params = [a.strip() for a in " ".join(args.split()).split(",")]
        params = [] if params == ["void"] else params
        out[name] = (_letter(ret), "".join(_letter(p.rsplit(" ", 1)[0]) for p in params))
    return out


def test_companion_header_builds_on_the_main_one():
    text = open(HEADER).read()
    assert '#include "metrics_b200.h"' in text
    main = open(os.path.join(ROOT, "include", "metrics_b200.h")).read()
    assert not set(_header_signatures()) & set(re.findall(r"MB200_API[^;(]*?\b(mb200_\w+)\s*\(", main))


def test_calibration_table_matches_the_header_and_the_library_exports_it():
    from metrics_b200 import _native

    assert _native.CALIBRATION_SIGNATURES == _header_signatures()
    assert len(_native.CALIBRATION_SIGNATURES) == 4
    raw = ctypes.CDLL(_native.lib_path())
    missing = [n for n in _native.CALIBRATION_SIGNATURES if not hasattr(raw, n)]
    assert not missing, missing
    handle = _native.lib()
    for name, (ret, args) in _native.CALIBRATION_SIGNATURES.items():
        fn = getattr(handle, name)
        assert fn.restype is _native._C_TYPES[ret] and len(fn.argtypes) == len(args), name
    assert handle.mb200_abi_version() == 1


class _RecordingLibrary:
    """Every calibration entry point as a real ctypes function pointer with the declared signature around a recorder."""

    def __init__(self, native):
        self.calls = {}
        self._keep = []
        for name, (ret, args) in native.CALIBRATION_SIGNATURES.items():
            proto = ctypes.CFUNCTYPE(native._C_TYPES[ret], *[native._C_TYPES[a] for a in args])

            def callback(*values, _name=name):
                self.calls.setdefault(_name, []).append(values)
                return 256 if _name.endswith("_bytes") else 0

            fn = proto(callback)
            self._keep.append(fn)
            setattr(self, name, fn)


def _patch_host(monkeypatch, native, stream):
    cpu = torch.device("cpu")
    monkeypatch.setattr(native, "require_cuda", lambda *t: cpu)
    monkeypatch.setattr(native, "on_device", lambda d: native._NOOP)
    monkeypatch.setattr(native, "stream_handle", lambda d: stream)


def test_every_calibration_wrapper_calls_the_abi_as_declared(monkeypatch):
    from metrics_b200 import _native

    fake = _RecordingLibrary(_native)
    monkeypatch.setattr(_native, "lib", lambda: fake)
    _patch_host(monkeypatch, _native, 0xABCD)
    scores, labels = torch.rand(16, 3), torch.randint(3, (16,))
    flag = torch.zeros(1, dtype=torch.int32)
    _native.calibration_top_label(scores, labels)
    _native.calibration_top_label(scores.double(), labels.int(), -1, flag)
    _native.calibration_bin_sums(scores[:, 0], labels, torch.linspace(0, 1, 16))
    assert set(fake.calls) == set(_native.CALIBRATION_SIGNATURES)
    for name, calls in fake.calls.items():
        args = _native.CALIBRATION_SIGNATURES[name][1]
        for values in calls:
            assert len(values) == len(args)
            if args.endswith("p"):
                assert values[-1] == 0xABCD, f"{name}: stream handle is not the last argument"
                assert values[0] not in (None, 0), f"{name}: first pointer is NULL"
    plain, checked = fake.calls["mb200_calibration_top_label"]
    assert plain[1] == _native.F32 and checked[1] == _native.F64 and checked[3] == _native.I32
    assert (plain[4], plain[5]) == (16, 3)
    assert plain[6] == 0 and checked[6] == 1 and checked[7] == -1
    assert plain[12] in (None, 0) and checked[12] not in (None, 0)
    bins = fake.calls["mb200_calibration_bin_sums"][0]
    assert bins[4] == 16 and bins[6] == 15 and bins[1] == _native.F32 and bins[3] == _native.I64


def test_real_library_accepts_the_calibration_wrappers_arguments_up_to_the_first_cuda_call(monkeypatch):
    """GPU-less boxes only: argument conversion and the library's own checks pass, the first failure is a CUDA error."""
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present: host pointers must not reach the kernels")
    from metrics_b200 import _native

    _patch_host(monkeypatch, _native, 0)
    scores, labels = torch.rand(16, 3), torch.randint(3, (16,))
    calls = {
        "top_label": lambda: _native.calibration_top_label(scores, labels, -1, torch.zeros(1, dtype=torch.int32)),
        "top_label_wide": lambda: _native.calibration_top_label(torch.rand(4, 1500), labels[:4]),
        "top_label_f64": lambda: _native.calibration_top_label(scores.double(), labels),
        "bin_sums": lambda: _native.calibration_bin_sums(scores[:, 0], labels, torch.linspace(0, 1, 16)),
        "bin_sums_f16": lambda: _native.calibration_bin_sums(scores[:, 0].half(), labels.bool(), torch.linspace(0, 1, 101).half()),
    }
    for name, call in calls.items():
        with pytest.raises(_native.NativeLibraryError, match=r"\(code -2\): CUDA error"):
            call()


def test_library_rejects_bad_calibration_arguments(monkeypatch):
    """Argument errors are ValueErrors raised before any CUDA call (works with and without a device: host tensors)."""
    from metrics_b200 import _native

    _patch_host(monkeypatch, _native, 0)
    with pytest.raises(ValueError, match="n_bins must lie in"):
        _native.calibration_bin_sums(torch.rand(4), torch.ones(4), torch.linspace(0, 1, 9000))
    with pytest.raises(ValueError, match="preds must be"):
        _native.calibration_top_label(torch.randint(3, (4, 3)), torch.zeros(4, dtype=torch.long))
    with pytest.raises(ValueError, match="target must be an integer"):
        _native.calibration_top_label(torch.rand(4, 3), torch.zeros(4))
