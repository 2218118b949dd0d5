"""Hausdorff distance for semantic segmentation (reference: functional/segmentation/hausdorff_distance.py).

One call of kernel K19 replaces the reference's Python loop over every (sample, class) pair, its binary erosion and its
dense distance transforms; one host synchronisation, the read of the kernel's error word, raises the reference's errors
at the update that met them.  2-D images only, as in the reference; unlike the reference, non-square images get the true
distance (DESIGN.md K19)."""
from __future__ import annotations

from typing import Optional, Union

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200 import _native
from metrics_b200.functional.segmentation.utils import _FLOAT_NAME, _raise_label_errors
from metrics_b200.utilities.checks import _check_same_shape

_EMPTY_MAX = ("max(): Expected reduction dim to be specified for input.numel() == 0. Specify the reduction dim with the "
              "'dim' argument.")


def _hausdorff_distance_validate_args(
    num_classes: int,
    include_background: bool,
    distance_metric: Literal["euclidean", "chessboard", "taxicab"] = "euclidean",
    spacing: Optional[Union[Tensor, list[float]]] = None,
    directed: bool = False,
    input_format: Literal["one-hot", "index"] = "one-hot",
) -> None:
    """Validate the arguments of `hausdorff_distance` function."""
    if num_classes <= 0:
        raise ValueError(f"Expected argument `num_classes` must be a positive integer, but got {num_classes}.")
    if not isinstance(include_background, bool):
        raise ValueError(f"Expected argument `include_background` must be a boolean, but got {include_background}.")
    if distance_metric not in ["euclidean", "chessboard", "taxicab"]:
        raise ValueError(
            f"Arg `distance_metric` must be one of 'euclidean', 'chessboard', 'taxicab', but got {distance_metric}."
        )
    if spacing is not None and not isinstance(spacing, (list, Tensor)):
        raise ValueError(f"Arg `spacing` must be a list or tensor, but got {type(spacing)}.")
    if not isinstance(directed, bool):
        raise ValueError(f"Expected argument `directed` must be a boolean, but got {directed}.")
    if input_format not in ["one-hot", "index"]:
        raise ValueError(f"Expected argument `input_format` to be one of 'one-hot', 'index', but got {input_format}.")


def _check_inputs(preds: Tensor, target: Tensor, spacing, index: bool) -> list:
    """The errors the host knows before reading any data, raised up front in the order the reference meets them per
    pair: spatial rank, floating-point inputs, rank 3, then the spacing.  Returns the spacing as a two-entry list."""
    if index:
        for x in (preds, target):
            if x.dtype != torch.int64:
                raise RuntimeError("one_hot is only applicable to index tensor of type LongTensor.")
    rank = preds.ndim - (1 if index else 2)
    if rank not in (2, 3):
        raise ValueError(f"Expected argument `preds` to be of rank 2 or 3 but got rank `{rank}`.")
    if not index and (preds.is_floating_point() or target.is_floating_point()):
        dtype = torch.promote_types(preds.dtype, target.dtype)
        raise NotImplementedError(
            f"\"bitwise_or_{preds.device.type}\" not implemented for '{_FLOAT_NAME.get(dtype, dtype)}'"
        )
    if rank == 3:
        raise ValueError("Expected argument `x` to be of rank 2 but got rank `3`.")
    if spacing is None:
        return [1, 1]
    if not isinstance(spacing, list):
        raise ValueError(f"Expected argument `sampling` to either be `None` or of type `list` but got `{type(spacing)}`.")
    if len(spacing) != 2:
        raise ValueError(f"Expected argument `sampling` to have length 2 but got length `{len(spacing)}`.")
    return [v if isinstance(v, int) else float(v) for v in spacing]


def hausdorff_distance(
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    include_background: bool = False,
    distance_metric: Literal["euclidean", "chessboard", "taxicab"] = "euclidean",
    spacing: Optional[Union[Tensor, list[float]]] = None,
    directed: bool = False,
    input_format: Literal["one-hot", "index"] = "one-hot",
) -> Tensor:
    """Hausdorff distance of every sample and class, float32 ``[N, C']`` on the inputs' device.

    ``preds`` / ``target``: one-hot ``(N, C, H, W)`` bool or integer tensors (dtypes may differ; any strides), or int64
    class indices ``(N, H, W)`` with ``input_format="index"``; CUDA tensors.  ``spacing``: two entries, pixel spacing
    along H and W (an int entry is int64 arithmetic, a float entry float32, as in the reference)."""
    _hausdorff_distance_validate_args(num_classes, include_background, distance_metric, spacing, directed, input_format)
    _check_same_shape(preds, target)
    index = input_format == "index"
    sampling = _check_inputs(preds, target, spacing, index)
    n = preds.shape[0]
    c = num_classes if index else preds.shape[1]
    cp = c - 1 if not include_background and c > 1 else c
    if n == 0 or cp == 0:
        return torch.zeros(n, cp, device=preds.device)
    if preds.shape[-2] * preds.shape[-1] == 0:  # every mask is empty: the first pair raises
        raise RuntimeError(_EMPTY_MAX)
    out, err = _native.hausdorff_distance(preds, target, num_classes, index, not include_background, distance_metric,
                                          sampling, directed)
    code, labels = err.tolist()
    _raise_label_errors(labels)
    if code >= 0:
        if code % 4 == _native.HD_NO_EDGES:
            raise RuntimeError(_EMPTY_MAX)
        raise ValueError("Input x should be binarized")
    return out
