"""CPU: the retrieval C-ABI (include/metrics_b200_retrieval.h): the size guard; metric-kind rejection before any launch; CPU
tensors rejected.  Its signatures and constants are checked in tests/test_abi.py, its dtype tags in
tests/test_dtype_dispatch_abi.py."""
import pytest
import torch


def test_size_guard_is_the_scratch_query():
    from metrics_b200 import _native

    lib = _native.lib()
    assert lib.mb200_retrieval_sort_scratch_bytes(_native.RET_MAX_ELEMENTS, 4) > 0
    assert lib.mb200_retrieval_sort_scratch_bytes(_native.RET_MAX_ELEMENTS + 1, 0) == -1
    assert lib.mb200_retrieval_ideal_scratch_bytes(_native.RET_MAX_ELEMENTS + 1, 0) == -1
    assert lib.mb200_retrieval_evaluate_scratch_bytes(_native.RET_MAX_ELEMENTS + 1) == -1
    with pytest.raises(ValueError, match=r"at most 2\^30 - 1"):
        _native.retrieval_sort_scratch_bytes(1 << 30, 0)
    # the wide-index path needs room for two sorts
    assert lib.mb200_retrieval_sort_scratch_bytes(1000, 8) > lib.mb200_retrieval_sort_scratch_bytes(1000, 4)


def test_rejected_target_tag_fails_before_any_launch():
    """The group sort's target tags are checked in tests/test_dtype_dispatch_abi.py; here the metric kind of the evaluation."""
    from metrics_b200 import _native

    lib = _native.lib()
    before = lib.mb200_launch_count()
    assert lib.mb200_retrieval_evaluate(8, 8, None, 8, 8, 4, 9, 0, 0, 8, 8, 8, 1 << 20, None) == -1
    assert lib.mb200_retrieval_evaluate(8, 8, None, 8, 8, 4, _native.RET_NDCG, 0, 0, 8, 8, 8, 1 << 20, None) == -1
    assert lib.mb200_launch_count() == before


def test_wrappers_require_cuda_tensors():
    from metrics_b200 import _native
    from metrics_b200.functional.retrieval import retrieval_average_precision

    with pytest.raises(_native.NativeLibraryError, match="no CPU fallback"):
        retrieval_average_precision(torch.rand(5), torch.tensor([0, 1, 0, 1, 1]))
