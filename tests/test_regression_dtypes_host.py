"""CPU: the regression functionals on mixed-dtype, N-d and non-dividing `num_outputs` inputs against goldens from the
reference, with the kernel replaced by its stand-in (the GPU twin is in test_regression_paths_gpu.py)."""
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLDEN_DIR
from tests.regression_dtype_cases import replay


@pytest.fixture(scope="module")
def golden_reg_dtypes():
    return np.load(os.path.join(GOLDEN_DIR, "regression_dtypes.npz"), allow_pickle=False)


def test_replay_reference_goldens(golden_reg_dtypes, cpu_kernel_standins):
    assert replay(golden_reg_dtypes, "cpu") == int(golden_reg_dtypes["n_cases"]) > 100


def test_num_outputs_must_divide_the_element_count(cpu_kernel_standins):
    from metrics_b200 import _native

    with pytest.raises(ValueError, match="num_outputs=3"):
        _native.regression_sums(torch.zeros(10, 4), torch.zeros(10, 4), _native.REG_MSE, 3)


def test_compute_dtype_is_the_promoted_floating_dtype():
    from metrics_b200._native import regression_compute_dtype as cd

    x = lambda dtype: torch.zeros(2, dtype=dtype)  # noqa: E731
    assert cd(x(torch.float16), x(torch.float32)) == torch.float32
    assert cd(x(torch.float32), x(torch.bfloat16)) == torch.float32
    assert cd(x(torch.float16), x(torch.bfloat16)) == torch.float32
    assert cd(x(torch.float32), x(torch.float64)) == torch.float64
    assert cd(x(torch.int64), x(torch.float16)) == torch.float16
    assert cd(x(torch.int64), x(torch.int32)) == torch.float32
    assert cd(x(torch.bfloat16), x(torch.bfloat16)) == torch.bfloat16
