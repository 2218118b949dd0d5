"""CPU: the rank-correlation C-ABI (include/metrics_b200_rankcorr.h): the size guard; variant, alternative and scratch rejection
before any launch; the reference's argument and input errors; CPU tensors rejected.  Its signatures and constants are checked
in tests/test_abi.py, its dtype tags in tests/test_dtype_dispatch_abi.py."""
import pytest
import torch

from tests import rankcorr_cases as rcc


def test_size_guard_is_the_scratch_query():
    from metrics_b200 import _native

    lib = _native.lib()
    assert lib.mb200_rankcorr_scratch_bytes(_native.RANKCORR_MAX_ROWS, 1, 1) > 0
    assert lib.mb200_rankcorr_scratch_bytes(_native.RANKCORR_MAX_ROWS + 1, 1, 0) == -1
    assert lib.mb200_rankcorr_scratch_bytes(10, 0, 0) == -1
    assert lib.mb200_rankcorr_scratch_bytes(1000, 3, 1) > lib.mb200_rankcorr_scratch_bytes(1000, 3, 0)
    with pytest.raises(ValueError, match=r"at most 2\^30 - 1"):
        _native.rankcorr_scratch_bytes(1 << 30, 1, True)


def test_rejected_arguments_fail_before_any_launch():
    from metrics_b200 import _native

    lib = _native.lib()
    before = lib.mb200_launch_count()
    assert lib.mb200_kendall_rank_corrcoef(8, _native.F32, 8, _native.F32, 4, 1, 3, 0, 8, _native.F32, None, 8, 1 << 20, None, None) == -1
    assert lib.mb200_kendall_rank_corrcoef(8, _native.F32, 8, _native.F32, 4, 1, 1, 4, 8, _native.F32, 8, 8, 1 << 20, None, None) == -1
    assert lib.mb200_kendall_rank_corrcoef(8, _native.F32, 8, _native.F32, 4, 1, 1, 1, 8, _native.F32, None, 8, 1 << 20, None, None) == -1
    assert lib.mb200_kendall_rank_corrcoef(8, _native.F32, 8, _native.F32, 4, 1, 1, 0, 8, _native.F32, None, 8, 16, None, None) == -1
    assert "scratch too small" in lib.mb200_last_error().decode()
    assert lib.mb200_launch_count() == before


def test_reference_errors():
    from metrics_b200.functional.regression import kendall_rank_corrcoef, spearman_corrcoef
    from metrics_b200.regression import KendallRankCorrCoef, SpearmanCorrCoef

    p4, t4 = torch.rand(4), torch.rand(4)
    calls = {
        "spearman/int_inputs": lambda: spearman_corrcoef(torch.arange(4), torch.arange(4)),
        "spearman/shape": lambda: spearman_corrcoef(p4, t4[:3]),
        "spearman/ndim": lambda: spearman_corrcoef(torch.rand(4, 2, 2), torch.rand(4, 2, 2)),
        "SpearmanCorrCoef/num_outputs": lambda: SpearmanCorrCoef(num_outputs=2).update(torch.rand(4, 3), torch.rand(4, 3)),
        "SpearmanCorrCoef/one_output_2d": lambda: SpearmanCorrCoef().update(torch.rand(4, 3), torch.rand(4, 3)),
        "kendall/shape": lambda: kendall_rank_corrcoef(p4, t4[:3]),
        "kendall/ndim": lambda: kendall_rank_corrcoef(torch.rand(4, 2, 2), torch.rand(4, 2, 2)),
        "kendall/variant": lambda: kendall_rank_corrcoef(p4, t4, variant="d"),
        "kendall/alternative": lambda: kendall_rank_corrcoef(p4, t4, t_test=True, alternative="both"),
        "kendall/t_test": lambda: kendall_rank_corrcoef(p4, t4, t_test=1),
        "kendall/alternative_none": lambda: kendall_rank_corrcoef(p4, t4, t_test=True, alternative=None),
        "KendallRankCorrCoef/variant": lambda: KendallRankCorrCoef(variant="x"),
        "KendallRankCorrCoef/t_test": lambda: KendallRankCorrCoef(t_test="yes"),
        "KendallRankCorrCoef/alternative_none": lambda: KendallRankCorrCoef(t_test=True, alternative=None),
        "KendallRankCorrCoef/alternative": lambda: KendallRankCorrCoef(t_test=True, alternative="more"),
        "KendallRankCorrCoef/num_outputs": lambda: KendallRankCorrCoef(num_outputs=2).update(torch.rand(4, 3), torch.rand(4, 3)),
    }
    want = rcc.errors(rcc.load())
    assert set(want) == set(calls)
    for name, fn in calls.items():
        with pytest.raises(Exception) as info:
            fn()
        assert [type(info.value).__name__, str(info.value)] == want[name], name


def test_cpu_tensors_are_rejected():
    from metrics_b200 import _native
    from metrics_b200.functional.regression import kendall_rank_corrcoef, spearman_corrcoef
    from metrics_b200.regression import KendallRankCorrCoef

    with pytest.raises(_native.NativeLibraryError, match="no CPU fallback"):
        spearman_corrcoef(torch.rand(5), torch.rand(5))
    with pytest.raises(_native.NativeLibraryError, match="no CPU fallback"):
        kendall_rank_corrcoef(torch.rand(5), torch.rand(5), t_test=True)
    m = KendallRankCorrCoef()
    m.update(torch.rand(5), torch.rand(5))
    with pytest.raises(_native.NativeLibraryError, match="no CPU fallback"):
        m.compute()
