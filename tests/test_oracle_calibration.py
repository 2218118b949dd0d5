"""CPU: the calibration oracles (oracle/calibration.py) against the reference's goldens (tests/golden/calibration.npz).

The op chain, run on CPU tensors, must reproduce the reference's states bit for bit; the float64 `ce_compute` must agree
with the reference's `compute()` within what the reference's state-dtype accumulation loses."""
import os

import numpy as np
import pytest
import torch

from oracle import calibration as oc
from tests.conftest import GOLDEN_DIR

DTYPES = {0: torch.float32, 1: torch.float16, 2: torch.bfloat16, 3: torch.float64}
# |reference - float64 oracle| allowed per state dtype: the reference sums its bins in that dtype
TOL = {torch.float32: 2e-5, torch.float16: 2e-2, torch.bfloat16: 1.5e-1, torch.float64: 1e-12}


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN_DIR, "calibration.npz"), allow_pickle=False)


def cases(golden):
    for k in range(int(golden["n_cases"])):
        key = f"case{k}"
        binary, n_batches, n_bins, ignore, num_classes, code = (int(v) for v in golden[f"{key}/meta"])
        dtype = DTYPES[code]
        batches = [(torch.from_numpy(golden[f"{key}/preds{b}"]).to(dtype), torch.from_numpy(golden[f"{key}/target{b}"]))
                   for b in range(n_batches)]
        yield key, dict(binary=bool(binary), batches=batches, n_bins=n_bins, ignore=None if ignore == -999 else ignore,
                        num_classes=num_classes, dtype=dtype)


def boundaries(n_bins, dtype):
    return torch.linspace(0, 1, n_bins + 1, dtype=dtype).double().numpy()


def test_golden_covers_what_it_should(golden):
    metas = [golden[f"case{k}/meta"] for k in range(int(golden["n_cases"]))]
    assert {int(m[4]) for m in metas if not m[0]} >= {2, 5, 1000}
    assert {int(m[2]) for m in metas} >= {1, 15, 100}
    assert {int(m[3]) for m in metas} >= {-999, -1, 0}
    assert {int(m[5]) for m in metas if m[0]} == {0, 1, 2, 3}
    assert any(m[1] > 1 for m in metas if m[0]) and any(m[1] > 1 for m in metas if not m[0])


def test_docstring_values(golden):
    np.testing.assert_allclose(golden["doc/binary"], [0.2900, 0.2918, 0.3167], atol=5e-5)
    np.testing.assert_allclose(golden["doc/multiclass"], [0.2000, 0.2082, 0.2333], atol=5e-5)
    p, t = np.array([0.25, 0.25, 0.55, 0.75, 0.75], np.float32), np.array([0, 0, 1, 1, 1])
    b = boundaries(2, torch.float32)
    np.testing.assert_allclose([oc.ce_compute(p, t, b, n) for n in ("l1", "l2", "max")], golden["doc/binary"], rtol=1e-6)


def test_chain_reproduces_the_reference_states(golden):
    for key, c in cases(golden):
        confs, accs = [], []
        for preds, target in c["batches"]:
            if c["binary"]:
                conf, acc = oc.binary_calibration_update_chain(preds, target, c["ignore"])
            else:
                conf, acc = oc.multiclass_calibration_update_chain(preds, target, c["num_classes"], c["ignore"])
            confs.append(conf)
            accs.append(acc)
        conf, acc = torch.cat(confs), torch.cat(accs)
        want_conf = golden[f"{key}/conf"]
        got = conf.float().numpy() if conf.dtype in (torch.float16, torch.bfloat16) else conf.numpy()
        assert np.array_equal(got, want_conf, equal_nan=True), key
        assert np.array_equal(acc.numpy(), golden[f"{key}/acc"]), key


def test_float64_oracle_matches_the_reference_compute(golden):
    for key, c in cases(golden):
        conf, acc = golden[f"{key}/conf"], golden[f"{key}/acc"]
        b = boundaries(c["n_bins"], c["dtype"])
        for norm in ("l1", "l2", "max"):
            got = oc.ce_compute(conf, acc, b, norm)
            assert abs(got - float(golden[f"{key}/{norm}"])) <= TOL[c["dtype"]], (key, norm, got, float(golden[f"{key}/{norm}"]))


def test_chain_compute_is_the_reference_compute(golden):
    for key, c in cases(golden):
        conf = torch.from_numpy(golden[f"{key}/conf"]).to(c["dtype"] if c["binary"] else torch.float32)
        acc = torch.from_numpy(golden[f"{key}/acc"])
        for norm in ("l1", "l2", "max"):
            got = oc.ce_compute_chain(conf, acc, c["n_bins"], norm).to(conf.dtype).float().numpy()
            assert np.array_equal(got, golden[f"{key}/{norm}"].astype(np.float32), equal_nan=True), (key, norm)


def test_l2_zero_and_nan_slot():
    assert oc.ce_compute(np.array([0.0, 0.0, 1.0, 1.0]), np.array([0, 0, 1, 1]), boundaries(4, torch.float32), "l2") == 0.0
    count, sum_conf, _ = oc.bin_sums(np.array([np.nan, 1.0, 0.5, 0.0]), np.zeros(4), boundaries(2, torch.float32))
    assert count.tolist() == [1, 1, 2] and np.isnan(sum_conf[2])
