"""The cases of tests/golden/segmentation.npz (written by tests/golden/make_golden_segmentation.py), rebuilt as tensors, and
a runner that replays one through this package's classes and functionals."""
from __future__ import annotations

import os

import numpy as np
import torch

from tests.conftest import GOLDEN_DIR

DTYPES = {0: torch.int64, 1: torch.bool, 2: torch.uint8, 3: torch.float32, 4: torch.float16, 5: torch.int32}
AVERAGES = ("micro", "macro", "weighted", "none", None)
WEIGHTS = ("square", "simple", "linear")


def load():
    return np.load(os.path.join(GOLDEN_DIR, "segmentation.npz"), allow_pickle=False)


def _layout(x: torch.Tensor, layout: int) -> torch.Tensor:
    """Channels-last cases were built as `one_hot(...).movedim(-1, 1)`: give the kernel that layout again."""
    return x.movedim(1, -1).contiguous().movedim(-1, 1) if layout == 1 else x


def cases(golden, device="cpu"):
    for k in range(int(golden["n_cases"])):
        key = f"case{k}"
        kind, index, c, bg, option, n_batches, code, layout = (int(v) for v in golden[f"{key}/meta"])
        dtype = DTYPES[code]
        batches = [tuple(_layout(torch.from_numpy(golden[f"{key}/{w}{b}"]).to(dtype), layout).to(device)
                         for w in ("preds", "target")) for b in range(n_batches)]
        yield key, dict(kind=kind, index=bool(index), num_classes=c, include_background=bool(bg), option=option,
                        batches=batches, dtype=dtype, layout=layout)


def build(case):
    """(metric instance, functional) for a case, from this package."""
    from metrics_b200 import segmentation as S  # noqa: N812
    from metrics_b200.functional import segmentation as F  # noqa: N812

    kw = dict(num_classes=case["num_classes"], include_background=case["include_background"],
              input_format="index" if case["index"] else "one-hot")
    opt = case["option"]
    if case["kind"] == 0:
        return S.MeanIoU(per_class=bool(opt), **kw), lambda p, t: F.mean_iou(p, t, per_class=bool(opt), **kw)
    if case["kind"] == 1:
        return (S.DiceScore(average=AVERAGES[opt], **kw),
                lambda p, t: F.dice_score(p, t, average=AVERAGES[opt], **kw))
    wt, pc = WEIGHTS[opt % 3], opt >= 3
    return (S.GeneralizedDiceScore(per_class=pc, weight_type=wt, **kw),
            lambda p, t: F.generalized_dice_score(p, t, per_class=pc, weight_type=wt, **kw))


def states(metric, kind):
    if kind == 0:
        return {"score": metric.score, "num_batches": metric.num_batches}
    if kind == 1:
        return {s: torch.cat(getattr(metric, s)) for s in ("numerator", "denominator", "support")}
    return {"score": metric.score, "samples": metric.samples}


def as_np(t: torch.Tensor) -> np.ndarray:
    t = t.detach().cpu()
    return t.float().numpy() if t.dtype in (torch.float16, torch.bfloat16) else t.numpy()


def check_case(golden, key, case, device, rtol=1e-6):
    """Replay a case through the class and the functional on `device`; integer states exact, float16 states exact,
    other floats within `rtol`."""
    metric, fn = build(case)
    metric = metric.to(device)
    for p, t in case["batches"]:
        metric.update(p, t)
    for name, got in states(metric, case["kind"]).items():
        want = golden[f"{key}/{name}"]
        got_np = as_np(got)
        assert got_np.shape == want.shape, (key, name, got_np.shape, want.shape)
        if not got.is_floating_point() or got.dtype == torch.float16:
            assert got_np.dtype == want.dtype or got.dtype == torch.float16, (key, name, got_np.dtype, want.dtype)
            assert np.array_equal(got_np, want), (key, name)
        else:
            np.testing.assert_allclose(got_np, want, rtol=rtol, atol=1e-7, err_msg=f"{key}/{name}")
    np.testing.assert_allclose(as_np(metric.compute()), golden[f"{key}/compute"], rtol=rtol, atol=1e-7, err_msg=key)
    np.testing.assert_allclose(as_np(fn(*case["batches"][0])), golden[f"{key}/functional"], rtol=rtol, atol=1e-7,
                               err_msg=key)
