"""CPU: the C-ABI of kernel K20 (include/mb200_image.h) — declarations, exports, constants and the ctypes table
`_native.IMAGE_SIGNATURES` — and its wrappers driven against REAL ctypes function pointers and against the real library up
to its first CUDA call, as tests/test_abi.py does for the include/metrics_b200*.h set."""
import ctypes
import os
import re

import pytest
import torch

from metrics_b200 import _native
from tests.test_abi import _header_signatures, _patch_host, _source

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "mb200_image.h")
STREAM = 0xCAFE


def test_signature_table_matches_the_header():
    assert '#include "metrics_b200.h"' in open(HEADER).read()
    assert _native.IMAGE_SIGNATURES == _header_signatures(HEADER)
    assert not set(_native.IMAGE_SIGNATURES) & set(_native.SIGNATURES)


def test_library_exports_and_binds_the_entry_points():
    raw = ctypes.CDLL(_native.lib_path())
    handle = _native.lib()
    for name, (ret, args) in _native.IMAGE_SIGNATURES.items():
        assert hasattr(raw, name), name
        fn = getattr(handle, name)
        assert fn.restype is _native._C_TYPES[ret] and len(fn.argtypes) == len(args), name


def test_header_constants_match_the_binding():
    found = {k: int(v) for k, v in re.findall(r"#define\s+MB200_(SSIM_\w+)\s+(\d+)\b", _source(HEADER))}
    assert found == {k: getattr(_native, k) for k in ("SSIM_RANGE", "SSIM_C1", "SSIM_C2", "SSIM_CONSTS", "SSIM_MAX_TAPS")}


def test_scratch_size_guard():
    lib = _native.lib()
    one = lib.mb200_ssim_scratch_bytes(_native.F32, 2, 3, 1, 64, 64, 1, 11, 11, 0, 5, 5)
    assert one >= 2 * 3 * 2 * 2 * 16  # one float64 pair per 32 x 32 tile
    assert lib.mb200_ssim_scratch_bytes(_native.F64, 2, 3, 1, 64, 64, 1, 11, 11, 0, 5, 5) > one  # 16-row tiles
    assert lib.mb200_ssim_scratch_bytes(_native.F32, 2, 3, 1, 4, 64, 1, 11, 11, 0, 5, 5) == -1  # reflect pad >= size
    assert lib.mb200_ssim_scratch_bytes(_native.F32, 2, 3, 1, 64, 64, 1, 11, 0, 0, 5, 5) == -1  # no taps
    assert lib.mb200_ssim_scratch_bytes(_native.F32, 2, 3, 1, 64, 64, 1, 200, 200, 0, 5, 5) == -1  # shared memory
    assert lib.mb200_ssim_scratch_bytes(_native.I64, 2, 3, 1, 64, 64, 1, 11, 11, 0, 5, 5) == -1


@pytest.mark.parametrize("b", [1 << 27, 3 << 26, 1 << 28])
def test_scratch_size_is_exact_past_two_gigabytes(b):
    """One float64 pair per tile plus the data-range partials: 2^27 tiles and more need 2 GB and more, which must not
    wrap in 32 bits."""
    assert _native.lib().mb200_ssim_scratch_bytes(_native.F32, b, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0) == b * 16 + 32768


def test_scratch_size_rejects_2_31_tiles():
    assert _native.lib().mb200_ssim_scratch_bytes(_native.F32, 1 << 31, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0) == -1


class _Recorder:
    def __init__(self):
        self.calls = {}
        for name, (ret, args) in _native.IMAGE_SIGNATURES.items():
            def callback(*values, _name=name):
                self.calls.setdefault(_name, []).append(values)
                return 4096 if _name.endswith("_bytes") else 0

            setattr(self, name, ctypes.CFUNCTYPE(_native._C_TYPES[ret], *[_native._C_TYPES[a] for a in args])(callback))


def _drive_ssim(data_range=None, clamp=None):
    p = torch.zeros(2, 3, 20, 24).contiguous(memory_format=torch.channels_last)
    t = torch.zeros(2, 3, 24, 20, dtype=torch.float64).transpose(2, 3)
    w = torch.ones(23)
    return p, t, _native.ssim(p, t, w, (1, 11, 11), (0, 5, 5), False, clamp, data_range, 0.01, 0.03, True, True)


def test_wrappers_call_the_abi_as_declared(monkeypatch):
    fake = _Recorder()
    monkeypatch.setattr(_native, "lib", lambda: fake)
    _patch_host(monkeypatch, STREAM)
    p, t, (sim, cs, img) = _drive_ssim()
    assert sim.shape == cs.shape == (2,) and sim.dtype == torch.float64 and img.shape == (2, 3, 1, 20, 24)
    (rng,) = fake.calls["mb200_ssim_data_range"]
    (upd,) = fake.calls["mb200_ssim_update"]
    for call, name in ((rng, "mb200_ssim_data_range"), (upd, "mb200_ssim_update")):
        assert len(call) == len(_native.IMAGE_SIGNATURES[name][1]) and call[-1] == STREAM
        assert call[1] == _native.F32 and call[3] == _native.F64 and call[4:9] == (2, 3, 1, 20, 24)
        assert call[9:14] == (p.stride(0), p.stride(1), 0, p.stride(2), p.stride(3))
        assert call[14:19] == (t.stride(0), t.stride(1), 0, t.stride(2), t.stride(3))
    assert rng[19:21] == (0.01, 0.03) and rng[22] is not None and rng[-2] == 4096
    assert upd[19:26] == (1, 11, 11, 0, 5, 5, 0) and upd[27] == 0  # taps, pads, no depth crop, no clamp
    assert upd[30] == rng[21] and all(upd[k] is not None for k in (26, 33, 34, 35, 36))  # consts of the pre-pass
    fake.calls.clear()
    _drive_ssim(data_range=0.5, clamp=(0.25, 0.75))
    assert "mb200_ssim_data_range" not in fake.calls
    (upd,) = fake.calls["mb200_ssim_update"]
    assert upd[27:33] == (1, 0.25, 0.75, None, (0.01 * 0.5) ** 2, (0.03 * 0.5) ** 2)
    po, to = _native.ssim_avg_pool(torch.zeros(2, 3, 9, 10, 11), torch.zeros(2, 3, 9, 10, 11).half(), True)
    (pool,) = fake.calls["mb200_ssim_avg_pool"]
    assert po.shape == to.shape == (2, 3, 4, 5, 5) and to.dtype == torch.float32
    assert pool[3] == _native.F16 and pool[4:9] == (2, 3, 9, 10, 11) and pool[19] == 1 and pool[-1] == STREAM


def test_real_library_accepts_every_wrappers_arguments_up_to_the_first_cuda_call(monkeypatch):
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present: host pointers must not reach the kernels")
    _patch_host(monkeypatch, 0)
    for drive in (lambda: _drive_ssim(), lambda: _drive_ssim(0.5, (0.25, 0.75)),
                  lambda: _native.ssim_avg_pool(torch.zeros(1, 1, 8, 8), torch.zeros(1, 1, 8, 8), False)):
        with pytest.raises(_native.NativeLibraryError, match=r"\(code -2\): CUDA error"):
            drive()


@pytest.mark.parametrize("bad", [-1, _native.I64, _native.I32, _native.U8, _native.BOOL, 10])
def test_library_rejects_non_float_dtype_tags_before_any_launch(bad):
    lib = _native.lib()
    geo = (1, 1, 1, 16, 16) + (256, 256, 0, 16, 1) * 2
    for which, msg in ((0, f"preds must be a floating-point tensor (dtype tag {bad})"),
                       (1, f"target must be a floating-point tensor (dtype tag {bad})")):
        tags = (bad, _native.F32) if which == 0 else (_native.F32, bad)
        for rc in (lib.mb200_ssim_update(8, tags[0], 8, tags[1], *geo, 1, 3, 3, 0, 1, 1, 0, 8, 0, 0.0, 0.0, None, 1.0, 1.0,
                                         8, None, None, 16, 1 << 20, None),
                   lib.mb200_ssim_data_range(8, tags[0], 8, tags[1], *geo, 0.01, 0.03, 8, 16, 1 << 20, None),
                   lib.mb200_ssim_avg_pool(8, tags[0], 8, tags[1], *geo, 0, 8, 8, None)):
            assert rc == -1 and lib.mb200_last_error().decode() == msg
