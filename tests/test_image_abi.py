"""CPU: the C-ABI of kernels K20 and K21 (include/metrics_b200_image.h): the scratch-size guard and the geometry checks
before any launch.  Their signatures, constants and argument passing are checked in tests/test_abi.py, their dtype tags in
tests/test_dtype_dispatch_abi.py."""
import pytest

from metrics_b200 import _native


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


def test_vif_and_uqi_reject_bad_geometry_before_any_launch():
    lib = _native.lib()
    geo = (1, 1, 1, 48, 48) + (2304, 2304, 0, 48, 1) * 2
    small = (1, 1, 1, 16, 16) + (256, 256, 0, 16, 1) * 2
    f = _native.F32
    checks = [
        (lambda: lib.mb200_vif_scale_update(8, f, 8, f, *geo, 1, 0, 17, 8, 1e-10, 2.0, 8, 8, 16, 1 << 20, None), "tap counts"),
        (lambda: lib.mb200_vif_scale_update(8, f, 8, f, *geo, 1, 256, 17, 8, 1e-10, 2.0, 8, 8, 16, 1 << 20, None), "tap counts"),
        (lambda: lib.mb200_vif_scale_update(8, f, 8, f, *small, 1, 17, 17, 8, 1e-10, 2.0, 8, 8, 16, 1 << 20, None), "empty output"),
        (lambda: lib.mb200_vif_decimate(8, f, 8, f, *small, 17, 9, 8, 8, 8, None), "empty output"),
        (lambda: lib.mb200_vif_decimate(8, f, 8, f, *geo, 0, 9, 8, 8, 8, None), "tap counts"),
        (lambda: lib.mb200_uqi_update(8, f, 8, f, *small, 1, 11, 11, 0, 16, 5, 5, 5, 8, 1e-7, 8, None, 16, 1 << 20, None),
         "reflect pads"),
        (lambda: lib.mb200_uqi_update(8, f, 8, f, *small, 1, 11, 11, 0, 5, 5, -1, 5, 8, 1e-7, 8, None, 16, 1 << 20, None),
         "crop margins"),
        (lambda: lib.mb200_uqi_update(8, f, 8, f, *small, 1, 41, 11, 0, 5, 5, 5, 5, 8, 1e-7, 8, None, 16, 1 << 20, None),
         "empty output"),
    ]
    for call, msg in checks:
        assert call() == -1 and msg in lib.mb200_last_error().decode(), msg
