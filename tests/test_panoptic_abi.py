"""CPU: the C-ABI of kernel K18 (include/mb200_panoptic.h) — declarations, exports and the ctypes table
`_native.PANOPTIC_SIGNATURES` — and its wrapper driven against a recording stand-in of the library, as tests/test_abi.py
does for the include/metrics_b200*.h entry points."""
import ctypes
import os
import re

import torch

from metrics_b200 import _native
from tests.test_abi import _header_signatures, _patch_host, _source

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "mb200_panoptic.h")
STREAM = 0xBEEF


def test_signature_table_matches_the_header():
    assert '#include "metrics_b200.h"' in open(HEADER).read()
    assert _native.PANOPTIC_SIGNATURES == _header_signatures(HEADER)
    assert not set(_native.PANOPTIC_SIGNATURES) & set(_native.SIGNATURES)


def test_library_exports_and_binds_the_entry_points():
    raw = ctypes.CDLL(_native.lib_path())
    handle = _native.lib()
    for name, (ret, args) in _native.PANOPTIC_SIGNATURES.items():
        assert hasattr(raw, name), name
        fn = getattr(handle, name)
        assert fn.restype is _native._C_TYPES[ret] and len(fn.argtypes) == len(args), name


def test_header_constants_match_the_binding():
    found = dict(re.findall(r"#define\s+MB200_(\w+)\s+(\d+)u\b", _source(HEADER)))
    assert {k: int(v) for k, v in found.items()} == {"PQ_UNKNOWN_PREDS": _native.PQ_UNKNOWN_PREDS,
                                                     "FLAG_CAPACITY": _native.FLAG_CAPACITY}


def test_scratch_size_guard():
    lib = _native.lib()
    ok = lib.mb200_panoptic_scratch_bytes(8, 1 << 21, 19, 8, 2048, 8192, _native.I64, _native.U8)
    assert ok > 8 * (2048 * 16 * 2 + 8192 * 16)
    assert lib.mb200_panoptic_scratch_bytes(8, 1 << 21, 19, 8, 3000, 8192, _native.I64, _native.I64) == -1  # not a power of 2
    assert lib.mb200_panoptic_scratch_bytes(8, 1 << 21, 19, 8, 2048, 8192, _native.F32, _native.I64) == -1
    assert lib.mb200_panoptic_scratch_bytes(8, 1 << 21, 19, 8, 2048, 8192, _native.I64, _native.BOOL) == -1
    assert lib.mb200_panoptic_scratch_bytes(8, (1 << 30) + 1, 19, 1, 2048, 8192, _native.I64, _native.I64) == -1


class _Recorder:
    """Real ctypes function pointers with the declared signatures around Python callbacks; the error word reads as
    `flags` so that the capacity repeat can be driven."""

    def __init__(self, flags):
        self.calls = {}
        self.flags = flags
        for name, (ret, args) in _native.PANOPTIC_SIGNATURES.items():
            def callback(*values, _name=name):
                self.calls.setdefault(_name, []).append(values)
                if _name.endswith("_bytes"):
                    return 1024
                ctypes.c_int32.from_address(values[20]).value = self.flags
                return 0

            setattr(self, name, ctypes.CFUNCTYPE(_native._C_TYPES[ret], *[_native._C_TYPES[a] for a in args])(callback))


def _drive(monkeypatch, flags, shape=(3, 5, 7, 2)):
    fake = _Recorder(flags)
    monkeypatch.setattr(_native, "lib", lambda: fake)
    _patch_host(monkeypatch, STREAM)
    states = (torch.zeros(4, dtype=torch.float64), *(torch.zeros(4, dtype=torch.int32) for _ in range(3)))
    preds = torch.zeros(shape, dtype=torch.int64)
    target = torch.zeros(shape, dtype=torch.uint8)
    cats = _native.panoptic_categories({1, 3}, {2, 9}, torch.device("cpu"))
    unknown = _native.panoptic_update_(*states, preds, target, cats, 2, True, False)
    return fake, unknown


def test_wrapper_calls_the_abi_as_declared(monkeypatch):
    fake, unknown = _drive(monkeypatch, 0)
    assert not unknown
    (call,) = fake.calls["mb200_panoptic_update"]
    assert len(call) == len(_native.PANOPTIC_SIGNATURES["mb200_panoptic_update"][1]) and call[-1] == STREAM
    assert call[1] == _native.I64 and call[3] == _native.U8 and call[4:6] == (3, 35)
    assert call[7:11] == (4, 2, 1, 0)  # categories, things, modified, allow_unknown_preds
    assert call[11:14] == (3, 128, 128)  # all images in one launch; tables no larger than 2 * pixels needs
    assert all(v not in (None, 0) for v in (call[0], call[2], call[6], *call[14:19], call[20]))


def test_capacity_flag_repeats_the_update_with_tables_that_cannot_fill(monkeypatch):
    fake, unknown = _drive(monkeypatch, _native.FLAG_CAPACITY, shape=(2, 64, 64, 2))
    first, again = fake.calls["mb200_panoptic_update"]
    assert first[12:14] == (2048, 8192) and again[12:14] == (8192, 8192) and not unknown


def test_unknown_preds_flag_is_reported_without_a_repeat(monkeypatch):
    fake, unknown = _drive(monkeypatch, _native.PQ_UNKNOWN_PREDS | _native.FLAG_CAPACITY)
    assert unknown and len(fake.calls["mb200_panoptic_update"]) == 1


def test_categories_table():
    cats = _native.panoptic_categories({7, 3}, {5, 1}, torch.device("cpu"))
    assert cats.tolist() == [1, 3, 5, 7, 2, 0, 3, 1]
