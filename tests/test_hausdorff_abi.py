"""CPU: the C-ABI of kernel K19 (include/metrics_b200_hausdorff.h): the scratch-size guard.  Its signatures, constants and
argument passing are checked in tests/test_abi.py."""
from metrics_b200 import _native


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
