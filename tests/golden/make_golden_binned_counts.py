"""Generate tests/golden/binned_counts.npz from the UNMODIFIED reference (TorchMetrics under /root/reference), CPU tensors.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_binned_counts.py

Same import set-up as make_golden.py.  Each set is one update of the reference's binned precision-recall-curve state
(`_*_precision_recall_curve_format` + `_*_update`): binary, multiclass, multiclass micro and multilabel, for every score dtype
(float16, bfloat16, float32, float64) and threshold kind (float16, bfloat16, float32, float64 and int64 tensors, a Python
list), with thresholds unsorted and duplicated, some not representable in the score dtype.  The binary, multiclass and micro
batches sit on either side of the reference's size rule (50 000 scores; N * C * C = 10^6), so both update branches are
pinned; those scores are not stored but regenerated from their seed by `oracle.binned_counts.scores_near`.  Multilabel sets
cover `ignore_index` None, 0, 1 and -1 on int64 targets, and 257, 0, 1 on uint8 targets, for which the reference raises (its
sentinel wraps in uint8); the golden records that it raised.  tests/test_oracle_binned_counts.py replays them through
oracle/binned_counts.py.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "_standins"))
sys.path.insert(0, "/root/reference/src")
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import torchmetrics.functional.classification.precision_recall_curve  # noqa: E402,F401
ref = sys.modules["torchmetrics.functional.classification.precision_recall_curve"]

from oracle.binned_counts import scores_near  # noqa: E402

SCORE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2, torch.float64: 3}
THR_KINDS = ["float16", "bfloat16", "float32", "float64", "int64", "list"]
# unsorted, 0.3 twice, values float16 / bfloat16 / float32 cannot hold, a float32 subnormal, -0
THR_VALUES = [0.5, 0.1, 0.9999, 0.3, 0.0, 1.0, 0.3, 0.7, 0.33333333, 0.9, 0.2, 1e-40, -0.0, 0.70000001]
INT_VALUES = [1, 0, 0, 2, -1]
C = 10


def thresholds(kind: str):
    if kind == "list":
        return list(THR_VALUES)
    if kind == "int64":
        return torch.tensor(INT_VALUES, dtype=torch.int64)
    return torch.tensor(THR_VALUES, dtype=torch.float64).to(getattr(torch, kind))


def points() -> torch.Tensor:
    return torch.tensor(THR_VALUES + INT_VALUES, dtype=torch.float64)


def main() -> None:
    out: dict = {}
    i = 0
    seed = 1000

    def add(task, dt, kind, n, state, extra=(0, 0, 0)):
        nonlocal i
        out[f"set{i}/meta"] = np.array([SCORE_CODE[dt], THR_KINDS.index(kind), n, seed, *extra], dtype=np.int64)
        out[f"set{i}/task"] = np.array(task)
        out[f"set{i}/state"] = state.numpy() if state is not None else np.zeros(0, dtype=np.int64)
        i += 1

    for dt in SCORE_CODE:
        for kind in THR_KINDS:
            # binary: on either side of 50 000 scores
            for n in (50_000, 50_001):
                seed += 1
                p = scores_near(points(), (n,), dt, seed)
                t = torch.randint(0, 2, (n,), generator=torch.Generator().manual_seed(seed))
                pf, tf, thr = ref._binary_precision_recall_curve_format(p, t, thresholds(kind))
                add("binary", dt, kind, n, ref._binary_precision_recall_curve_update(pf, tf, thr))
            # multiclass: N * C * C on either side of 10^6; micro: N * C on either side of 50 000
            for task, n in (("multiclass", 10_000), ("multiclass", 10_001), ("micro", 5_000), ("micro", 5_001)):
                seed += 1
                p = scores_near(points(), (n, C), dt, seed)
                t = torch.randint(0, C, (n,), generator=torch.Generator().manual_seed(seed))
                avg = "micro" if task == "micro" else None
                pf, tf, thr = ref._multiclass_precision_recall_curve_format(p, t, C, thresholds(kind), None, avg)
                add(task, dt, kind, n, ref._multiclass_precision_recall_curve_update(pf, tf, C, thr, avg))
            # multilabel: ignore_index on int64 and uint8 targets
            for tdt, ign in ((torch.int64, None), (torch.int64, 0), (torch.int64, 1), (torch.int64, -1), (torch.uint8, 257),
                             (torch.uint8, 0), (torch.uint8, 1)):
                seed += 1
                n, lab = 40, 3
                p = scores_near(points(), (n, lab), dt, seed)
                t = torch.randint(0, 2, (n, lab), generator=torch.Generator().manual_seed(seed))
                if ign == -1:
                    t[::3, 1] = -1
                t = t.to(tdt)
                try:
                    pf, tf, thr = ref._multilabel_precision_recall_curve_format(p, t, lab, thresholds(kind), ign)
                    state = ref._multilabel_precision_recall_curve_update(pf, tf, lab, thr)
                except RuntimeError:
                    state = None  # the sentinel wrapped in uint8: reshape of a too-long bincount
                extra = (int(tdt == torch.uint8), ign is not None, ign if ign is not None else 0)
                add("multilabel", dt, kind, n, state, extra)
    out["n_sets"] = np.array(i)
    np.savez_compressed(os.path.join(HERE, "binned_counts.npz"), **out)
    print(f"wrote {i} sets")


if __name__ == "__main__":
    main()
