"""CPU: the C-ABI of kernel K18 (include/metrics_b200_panoptic.h): the scratch-size guard, the capacity repeat and the
unknown-preds report of the wrapper, and its categories table.  Its signatures, constants and argument passing are checked in
tests/test_abi.py."""
import torch

from metrics_b200 import _native
from tests.test_abi import _error_word, _panoptic_update, _patch_host, _Recorder

STREAM = 0xBEEF


def test_scratch_size_guard():
    lib = _native.lib()
    ok = lib.mb200_panoptic_scratch_bytes(8, 1 << 21, 19, 8, 2048, 8192, _native.I64, _native.U8)
    assert ok > 8 * (2048 * 16 * 2 + 8192 * 16)
    assert lib.mb200_panoptic_scratch_bytes(8, 1 << 21, 19, 8, 3000, 8192, _native.I64, _native.I64) == -1  # not a power of 2
    assert lib.mb200_panoptic_scratch_bytes(8, 1 << 21, 19, 8, 2048, 8192, _native.F32, _native.I64) == -1
    assert lib.mb200_panoptic_scratch_bytes(8, 1 << 21, 19, 8, 2048, 8192, _native.I64, _native.BOOL) == -1
    assert lib.mb200_panoptic_scratch_bytes(8, (1 << 30) + 1, 19, 1, 2048, 8192, _native.I64, _native.I64) == -1


def _drive(monkeypatch, flags, shape=(3, 5, 7, 2)):
    """The update's calls when its error word reads `flags`."""
    fake = _Recorder({"mb200_panoptic_update": _error_word(flags)})
    monkeypatch.setattr(_native, "lib", lambda: fake)
    _patch_host(monkeypatch, STREAM)
    unknown = _panoptic_update(shape)
    return fake.calls[None]["mb200_panoptic_update"], unknown


def test_capacity_flag_repeats_the_update_with_tables_that_cannot_fill(monkeypatch):
    (first, again), unknown = _drive(monkeypatch, _native.FLAG_CAPACITY, shape=(2, 64, 64, 2))
    assert first[12:14] == (2048, 8192) and again[12:14] == (8192, 8192) and not unknown


def test_unknown_preds_flag_is_reported_without_a_repeat(monkeypatch):
    calls, unknown = _drive(monkeypatch, _native.PQ_UNKNOWN_PREDS | _native.FLAG_CAPACITY)
    assert unknown and len(calls) == 1


def test_categories_table():
    cats = _native.panoptic_categories({7, 3}, {5, 1}, torch.device("cpu"))
    assert cats.tolist() == [1, 3, 5, 7, 2, 0, 3, 1]
