"""CPU: the C-ABI of kernel K19 (include/mb200_hausdorff.h) — declarations, exports and the ctypes table
`_native.HAUSDORFF_SIGNATURES` — and its wrapper driven against a recording stand-in of the library, as
tests/test_panoptic_abi.py does for K18."""
import ctypes
import os
import re

import torch

from metrics_b200 import _native
from tests.test_abi import _header_signatures, _patch_host, _source

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "mb200_hausdorff.h")
STREAM = 0xBEEF


def test_signature_table_matches_the_header():
    assert '#include "metrics_b200.h"' in open(HEADER).read()
    assert _native.HAUSDORFF_SIGNATURES == _header_signatures(HEADER)
    assert not set(_native.HAUSDORFF_SIGNATURES) & (set(_native.SIGNATURES) | set(_native.PANOPTIC_SIGNATURES))


def test_library_exports_and_binds_the_entry_points():
    raw = ctypes.CDLL(_native.lib_path())
    handle = _native.lib()
    for name, (ret, args) in _native.HAUSDORFF_SIGNATURES.items():
        assert hasattr(raw, name), name
        fn = getattr(handle, name)
        assert fn.restype is _native._C_TYPES[ret] and len(fn.argtypes) == len(args), name


def test_header_constants_match_the_binding():
    src = _source(HEADER)
    found = dict(re.findall(r"#define\s+MB200_HD_(\w+)\s+(\d+)u?\b", src))
    assert {k: int(v) for k, v in found.items()} == {
        "PREDS_NOT_BINARY": _native.HD_PREDS_NOT_BINARY, "TARGET_NOT_BINARY": _native.HD_TARGET_NOT_BINARY,
        "NO_EDGES": _native.HD_NO_EDGES, **{k.upper(): v for k, v in _native.HD_METRICS.items()}}


def test_scratch_size_guard():
    lib = _native.lib()
    one = lib.mb200_hausdorff_scratch_bytes(512, 512, 0, 1)
    assert one >= 512 * 512 * (1 + 2 * 2)  # edge bytes and two uint16 column distances
    assert lib.mb200_hausdorff_scratch_bytes(512, 512, 1, 1) < one
    assert lib.mb200_hausdorff_scratch_bytes(200, 512, 0, 1) < 200 * 512 * (1 + 2 * 2) + 64  # uint8 below 256 rows
    assert lib.mb200_hausdorff_scratch_bytes(70000, 3, 0, 1) >= 70000 * 3 * 9  # uint32 above 65535 rows
    assert lib.mb200_hausdorff_scratch_bytes(512, 512, 0, 8) >= 8 * (one - 16)
    assert lib.mb200_hausdorff_scratch_bytes(0, 512, 0, 1) == -1
    assert lib.mb200_hausdorff_scratch_bytes(512, 512, 0, 0) == -1


class _Recorder:
    def __init__(self):
        self.calls = {}
        for name, (ret, args) in _native.HAUSDORFF_SIGNATURES.items():
            def callback(*values, _name=name):
                self.calls.setdefault(_name, []).append(values)
                return 1000 * values[3] if _name.endswith("_bytes") else 0

            setattr(self, name, ctypes.CFUNCTYPE(_native._C_TYPES[ret], *[_native._C_TYPES[a] for a in args])(callback))


def test_wrapper_calls_the_abi_as_declared(monkeypatch):
    fake = _Recorder()
    monkeypatch.setattr(_native, "lib", lambda: fake)
    monkeypatch.setattr(_native, "HAUSDORFF_SCRATCH_BYTES", 4000)
    _patch_host(monkeypatch, STREAM)
    preds = torch.zeros(3, 4, 5, 7, dtype=torch.uint8).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    target = torch.zeros(3, 4, 5, 7, dtype=torch.int32)
    out, err = _native.hausdorff_distance(preds, target, 4, False, True, "taxicab", [2, 0.5], True)
    assert out.shape == (3, 3) and out.dtype == torch.float32 and err.shape == (2,) and err.dtype == torch.int64
    (call,) = fake.calls["mb200_hausdorff_distance"]
    assert len(call) == len(_native.HAUSDORFF_SIGNATURES["mb200_hausdorff_distance"][1]) and call[-1] == STREAM
    assert call[1] == _native.U8 and call[3] == _native.I32 and call[4:9] == (1, 3, 4, 5, 7)
    assert call[9:13] == preds.stride() and call[13:17] == target.stride()
    assert call[17:23] == (1, 2, 1, 2.0, 0.5, 1)  # drop background, taxicab, axis 0 int, spacing, directed
    assert call[23] == 4 and call[26] == 4000  # pairs per launch under the scratch cap, the scratch of that launch
    assert all(v not in (None, 0) for v in (call[0], call[2], call[24], call[25], call[27]))


def test_index_labels_pass_three_strides(monkeypatch):
    fake = _Recorder()
    monkeypatch.setattr(_native, "lib", lambda: fake)
    _patch_host(monkeypatch, STREAM)
    lab = torch.zeros(2, 9, 6, dtype=torch.int64).transpose(1, 2)
    _native.hausdorff_distance(lab, lab, 5, True, False, "euclidean", [1, 1], False)
    (call,) = fake.calls["mb200_hausdorff_distance"]
    assert call[4:9] == (0, 2, 5, 6, 9) and call[9:13] == (54, 0, 1, 6) and call[19] == 3 and call[23] == 10
