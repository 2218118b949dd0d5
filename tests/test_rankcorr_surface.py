"""CPU: the rank-correlation C-ABI (include/metrics_b200_rankcorr.h) and its ctypes table `_native.RANKCORR_SIGNATURES`; the
size guard; dtype rejection before any launch; the reference's argument and input errors; CPU tensors rejected."""
import ctypes
import os
import re

import pytest
import torch

from tests import rankcorr_cases as rcc
from tests.conftest import ROOT
from tests.test_calibration_abi import _letter

HEADER = os.path.join(ROOT, "include", "metrics_b200_rankcorr.h")


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
    assert _native.RANKCORR_SIGNATURES == _header_signatures()
    main = open(os.path.join(ROOT, "include", "metrics_b200.h")).read()
    assert not set(_header_signatures()) & set(re.findall(r"MB200_API[^;(]*?\b(mb200_\w+)\s*\(", main))
    raw = ctypes.CDLL(_native.lib_path())
    assert all(hasattr(raw, n) for n in _native.RANKCORR_SIGNATURES)
    for name, (ret, args) in _native.RANKCORR_SIGNATURES.items():
        fn = getattr(_native.lib(), name)
        assert fn.restype is _native._C_TYPES[ret] and len(fn.argtypes) == len(args), name
    defines = dict(re.findall(r"#define MB200_KENDALL_(\w+) (\d+)\n", open(HEADER).read()))
    assert {k: int(defines[k]) for k in ("A", "B", "C")} == {k.upper(): v for k, v in _native.KENDALL_VARIANT.items()}
    alts = {"ALT_NONE": None, "ALT_TWO_SIDED": "two-sided", "ALT_LESS": "less", "ALT_GREATER": "greater"}
    assert all(_native.KENDALL_ALTERNATIVE[v] == int(defines[k]) for k, v in alts.items())
    assert _native.lib().mb200_abi_version() == 1


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
    for tag in (-1, _native.I64, _native.I32, _native.U8, 10):  # Spearman: floating point only
        assert lib.mb200_spearman_corrcoef(8, tag, 8, _native.F32, 4, 1, 8, _native.F32, 1e-6, 8, 1 << 20, None, None) == -1
    assert "floating point" in lib.mb200_last_error().decode()
    for tag in (-1, _native.I16, _native.I8, _native.U8, _native.BOOL, 10):  # Kendall: float, int32, int64
        assert lib.mb200_kendall_rank_corrcoef(8, _native.F32, 8, tag, 4, 1, 1, 0, 8, _native.F32, None, 8, 1 << 20, None, None) == -1
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
