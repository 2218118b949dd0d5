"""The per-sample overlap counts that every segmentation metric here starts from (reference:
functional/segmentation/{mean_iou,dice,generalized_dice}.py, the `_update` halves up to their three `sum`s).

One call of kernel K15 replaces the reference's `one_hot(...).movedim(-1, 1)` of both label maps (index format),
`_ignore_background` and the three reductions over the spatial axes."""
from __future__ import annotations

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200 import _native
from metrics_b200.utilities.checks import _check_same_shape

_FLOAT_NAME = {torch.float32: "Float", torch.float16: "Half", torch.bfloat16: "BFloat16", torch.float64: "Double"}
_NEEDS_3D = "Expected both `preds` and `target` to have at least 3 dimensions, but got {}."


def _raise_label_errors(flag: int) -> None:
    """The first error `torch.nn.functional.one_hot` would raise: preds before target, negative before too large."""
    for negative, too_large in ((_native.SEG_PREDS_NEGATIVE, _native.SEG_PREDS_TOO_LARGE),
                                (_native.SEG_TARGET_NEGATIVE, _native.SEG_TARGET_TOO_LARGE)):
        if flag & negative:
            raise RuntimeError("Class values must be non-negative.")
        if flag & too_large:
            raise RuntimeError("Class values must be smaller than num_classes.")


def _overlap_counts(
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    include_background: bool,
    input_format: Literal["one-hot", "index"],
    product: Literal["and", "mul"],
) -> tuple[Tensor, Tensor, Tensor]:
    """``(intersection, pred_sum, target_sum)``, each ``[N, C']``: the sums over every spatial position of
    ``preds & target`` (``product="and"``) or ``preds * target``, of ``preds`` and of ``target``, in the reference's
    dtypes (int64 for index and integer one-hot inputs, the input dtype for floating one-hot inputs).

    Index format: one host synchronisation, to raise the reference's out-of-range error at the update that met it (the
    counts leave such labels out).  One-hot format: none."""
    _check_same_shape(preds, target)
    index = input_format == "index"
    if index:
        for x in (preds, target):
            if x.dtype != torch.int64:
                raise RuntimeError("one_hot is only applicable to index tensor of type LongTensor.")
    else:
        if preds.ndim < 3:
            raise ValueError(_NEEDS_3D.format(preds.ndim))
        if preds.is_floating_point() and product == "and":
            raise NotImplementedError(
                f"\"bitwise_and_{preds.device.type}\" not implemented for '{_FLOAT_NAME.get(preds.dtype, preds.dtype)}'"
            )
        if preds.dtype != target.dtype:
            raise TypeError(f"metrics_b200: one-hot preds and target must share a dtype, got {preds.dtype} and {target.dtype}")
    flag = torch.zeros(1, dtype=torch.int32, device=preds.device) if index else None
    counts = _native.segmentation_overlap_counts(preds, target, num_classes, index, product == "mul", not include_background,
                                                 flag)
    if index:
        _raise_label_errors(int(flag.item()))
        if preds.ndim < 2:
            raise ValueError(_NEEDS_3D.format(preds.ndim + 1))
    if counts.dtype == torch.float64:
        counts = counts.to(preds.dtype)
    return counts[0], counts[1], counts[2]
