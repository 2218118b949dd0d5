"""CPU: the kernel wrappers refuse host tensors, product code stays clear of the oracle, and the threshold sortedness cache
tells tensors apart.  The C-ABI itself is checked in tests/test_abi.py."""
import os
import re

from tests.conftest import ROOT


def test_cpu_tensors_are_rejected_loudly():
    import pytest
    import torch

    from metrics_b200.classification import MulticlassConfusionMatrix
    from metrics_b200._native import NativeLibraryError

    m = MulticlassConfusionMatrix(num_classes=3, validate_args=False)
    with pytest.raises(NativeLibraryError, match="no CPU fallback"):
        m.update(torch.randn(4, 3), torch.tensor([0, 1, 2, 0]))


def test_product_never_imports_the_oracle():
    bad = []
    for dirpath, _, files in os.walk(os.path.join(ROOT, "metrics_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f), errors="replace").read()
                if re.search(r"^\s*(from|import)\s+(oracle|tests)\b", src, re.M) or "cpu_kernels" in src:
                    bad.append(os.path.join(dirpath, f))
    assert not bad, f"product code must not import oracle/ or the test stand-ins: {bad}"


def test_threshold_sortedness_is_not_shared_between_tensors_at_one_address():
    """Two views that start at the same address with the same length and version counter hold different thresholds."""
    import torch

    from metrics_b200 import _native

    x = torch.tensor([0.1, 0.05, 0.5])
    ascending, descending = x[::2], x[:2]
    assert ascending.data_ptr() == descending.data_ptr() and ascending._version == descending._version
    assert _native._is_sorted(ascending) and not _native._is_sorted(descending)
    x[2] = 0.0  # an in-place change is a new version
    assert not _native._is_sorted(ascending)
