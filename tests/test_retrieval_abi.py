"""CPU: the retrieval C-ABI (include/metrics_b200_retrieval.h) and its ctypes table `_native.RETRIEVAL_SIGNATURES`, checked
the way tests/test_segmentation_abi.py checks the segmentation header; the size guard; tag rejection before any launch."""
import ctypes
import os
import re

import pytest
import torch

from tests.conftest import ROOT
from tests.test_calibration_abi import _letter

HEADER = os.path.join(ROOT, "include", "metrics_b200_retrieval.h")


def _header_signatures():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    out = {}
    for ret, name, args in re.findall(r"MB200_API\s+([\w\s\*]+?)\s*(mb200_\w+)\s*\(([^)]*)\)\s*;", text):
        params = [a.strip() for a in " ".join(args.split()).split(",")]
        out[name] = (_letter(ret), "".join(_letter(p.rsplit(" ", 1)[0]) for p in params))
    return out


def test_table_matches_the_header_and_the_library_exports_it():
    from metrics_b200 import _native

    assert '#include "metrics_b200.h"' in open(HEADER).read()
    assert _native.RETRIEVAL_SIGNATURES == _header_signatures()
    main = open(os.path.join(ROOT, "include", "metrics_b200.h")).read()
    assert not set(_header_signatures()) & set(re.findall(r"MB200_API[^;(]*?\b(mb200_\w+)\s*\(", main))
    raw = ctypes.CDLL(_native.lib_path())
    assert all(hasattr(raw, n) for n in _native.RETRIEVAL_SIGNATURES)
    for name, (ret, args) in _native.RETRIEVAL_SIGNATURES.items():
        fn = getattr(_native.lib(), name)
        assert fn.restype is _native._C_TYPES[ret] and len(fn.argtypes) == len(args), name
    kinds = dict(re.findall(r"#define MB200_RET_(\w+) (\d+)\n", open(HEADER).read()))
    assert [int(kinds[k]) for k in ("AP", "RR", "PRECISION", "RECALL", "HIT_RATE", "FALL_OUT", "R_PRECISION", "NDCG")] == list(range(8))
    assert _native.lib().mb200_abi_version() == 1


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
    from metrics_b200 import _native

    lib = _native.lib()
    for tag in range(-1, 11):
        if tag in (_native.I64, _native.F32):
            continue
        before = lib.mb200_launch_count()
        rc = lib.mb200_retrieval_sort(8, 8, 8, tag, 4, 0, 0, 8, 8, 8, 8, 8, 1 << 20, None)
        assert rc == -1 and lib.mb200_launch_count() == before, tag
        assert lib.mb200_last_error().decode() == f"target must be int64 or float32 (dtype tag {tag})"
    before = lib.mb200_launch_count()
    assert lib.mb200_retrieval_evaluate(8, 8, None, 8, 8, 4, 9, 0, 0, 8, 8, 8, 1 << 20, None) == -1
    assert lib.mb200_retrieval_evaluate(8, 8, None, 8, 8, 4, _native.RET_NDCG, 0, 0, 8, 8, 8, 1 << 20, None) == -1
    assert lib.mb200_launch_count() == before


def test_wrappers_require_cuda_tensors():
    from metrics_b200 import _native
    from metrics_b200.functional.retrieval import retrieval_average_precision

    with pytest.raises(_native.NativeLibraryError, match="no CPU fallback"):
        retrieval_average_precision(torch.rand(5), torch.tensor([0, 1, 0, 1, 1]))
