"""CPU: the kernels convert score values, build descending sort keys and reduce warps through the one set of helpers in
metrics_b200/csrc/common.cuh, not through a copy per kernel file.

Each copy used to encode a rule the parity suites depend on (half / bfloat16 widen exactly, float64 is compared as
float32, results are stored in T with round-to-nearest, the descending key is ~f32_order_key with NaN first), so a copy
that drifts changes results in one kernel family only.  This scans every metrics_b200/csrc/*.cu for the removed copies."""
import glob
import os
import re

from tests.conftest import ROOT

CSRC = os.path.join(ROOT, "metrics_b200", "csrc")

# helpers common.cuh provides, and the per-file names they replace
SHARED = ["widen", "to_f32", "narrow", "round_to", "load_f64", "f32_desc_key", "warp_sum", "warp_max"]
REMOVED = ["to_float", "from_float", "score_to_float", "binned_to_float", "fz_to_float", "fz_from_float", "peer_to_float",
           "kl_load", "kl_store", "load_as_double", "binned_load", "binned_threshold", "load_value", "desc_key",
           "peer_desc_key", "score_key", "to_a", "from_f", "from_a"]
REMOVED_TYPES = ["Cal", "CmpType"]

# The half / bfloat16 intrinsics outside common.cuh, per file, where the arithmetic is the file's own:
#   binary.cu        host threshold_in_dtype / next_in_dtype (the scalar threshold in the score dtype, and its successor)
#   segmentation.cu  OH<__half>::prod / OH<__nv_bfloat16>::prod (the product with one rounding to T)
#   rankcorr.cu      order_key(__nv_bfloat16) (16-bit keys)
HALF_INTRINSICS = re.compile(r"\b(__half2float|__bfloat162float|__float2half_rn|__float2bfloat16_rn)\b")
HALF_INTRINSIC_LINES = {"binary.cu": 6, "segmentation.cu": 2, "rankcorr.cu": 1}


def _sources():
    paths = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
    assert len(paths) >= 18, paths
    out = {}
    for path in paths:
        text = re.sub(r"/\*.*?\*/", "", open(path).read(), flags=re.S)
        out[os.path.basename(path)] = re.sub(r"//[^\n]*", "", text)
    return out


def _defines(src, name):
    """True when `src` declares or defines a device function `name` (free, specialised or a static member)."""
    return re.search(r"\b__device__\b[^;{}]*?\b%s\s*(<[^<>;{}]*>)?\s*\(" % re.escape(name), src) is not None


def test_count_launch_is_declared_once_in_common():
    assert re.search(r"^void count_launch\(\);", open(os.path.join(CSRC, "common.cuh")).read(), flags=re.M)
    redeclared = [f for f, src in _sources().items() if re.search(r"\bextern\s+void\s+count_launch\b", src)]
    assert redeclared == []


def test_no_kernel_file_defines_its_own_conversion_key_or_warp_helper():
    copies = [(f, name) for f, src in _sources().items() for name in SHARED + REMOVED if _defines(src, name)]
    copies += [(f, name) for f, src in _sources().items() for name in REMOVED_TYPES
               if re.search(r"\bstruct\s+%s\b" % name, src)]
    assert copies == []


def test_half_intrinsics_only_where_the_arithmetic_is_the_files_own():
    found = {}
    for f, src in _sources().items():
        n = sum(1 for line in src.splitlines() if HALF_INTRINSICS.search(line))
        if n:
            found[f] = n
    assert found == HALF_INTRINSIC_LINES


def test_the_detector_sees_a_local_copy():
    copy = "template <>\n__device__ __forceinline__ float to_float<__half>(__half x) { return __half2float(x); }\n"
    member = "struct Cvt<float> {\n    __device__ static float to_a(float v) { return v; }\n};\n"
    assert _defines(copy, "to_float") and _defines(member, "to_a")
    assert not _defines("    const float v = to_f32(x);\n", "to_f32")
    assert not _defines("__device__ __forceinline__ bool f(T x) { return widen(x) > 0.f; }\n", "widen")
