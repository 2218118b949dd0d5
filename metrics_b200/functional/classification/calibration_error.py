"""Top-label calibration error (reference: functional/classification/calibration_error.py) on kernels K14a / K14b.

Update: the binary state is the reference's ``(preds, target)`` after flatten, ignore drop and ``sigmoid_if_logits`` (K6);
the multiclass state is ``(confidence, accuracy)`` from ONE read of the ``[N, C]`` scores (K14a: batch-global logits vote
without a host sync, row softmax, max / argmax over the softmax rounded to the input dtype, compare against the target).
Compute: exact counts and float64 sums per bin (K14b), rounded to the state dtype, then the reference's epilogue in ATen
ops.  The reference accumulates its bins in the state dtype, so its float32 counts stop growing at 2**24 samples per bin
(2048 / 256 for float16 / bfloat16 scores); here they do not (DESIGN.md, K14).
"""
from __future__ import annotations

from typing import Optional, Union

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200 import _native
from metrics_b200.functional.classification._validation import check_multiclass_shapes, new_flag, raise_if_flagged
from metrics_b200.utilities.checks import _check_same_shape
from metrics_b200.utilities.enums import ClassificationTaskNoMultilabel


def _epilogue_dtype(dtype: torch.dtype) -> torch.dtype:
    """float16 cannot hold a bin count above 65504: its epilogue runs in float32 and the result is rounded back."""
    return torch.float32 if dtype == torch.float16 else dtype


def _binning_bucketize(
    confidences: Tensor, accuracies: Tensor, bin_boundaries: Tensor
) -> tuple[Tensor, Tensor, Tensor]:
    """Binned accuracy, binned confidence and bin proportions (reference :30-61).

    The slot of a confidence is ``bucketize(confidences, bin_boundaries, right=True) - 1``, compared in the confidence
    dtype (kernel K14b).  Counts are exact and the sums are float64; they are rounded to the confidence dtype (float32 for
    float16) before the reference's divisions."""
    bin_boundaries = bin_boundaries.to(device=confidences.device, dtype=confidences.dtype)
    count, sum_conf, sum_acc = _native.calibration_bin_sums(confidences, accuracies, bin_boundaries)
    dtype = _epilogue_dtype(confidences.dtype)
    count_bin = count.to(dtype)
    conf_bin = torch.nan_to_num(sum_conf.to(dtype) / count_bin)
    acc_bin = torch.nan_to_num(sum_acc.to(dtype) / count_bin)
    prop_bin = count_bin / count_bin.sum()
    return acc_bin, conf_bin, prop_bin


def _ce_compute(
    confidences: Tensor,
    accuracies: Tensor,
    bin_boundaries: Union[Tensor, int],
    norm: str = "l1",
    debias: bool = False,
) -> Tensor:
    """Calibration error of the given confidences / accuracies under the given bin boundaries and norm (reference
    :64-113): l1 = ECE, max = MCE, l2 = RMSCE (optionally debiased).  ``tensor(0)`` when the l2 sum is not positive."""
    if isinstance(bin_boundaries, int):
        bin_boundaries = torch.linspace(0, 1, bin_boundaries + 1, dtype=confidences.dtype, device=confidences.device)

    if norm not in {"l1", "l2", "max"}:
        raise ValueError(f"Argument `norm` is expected to be one of 'l1', 'l2', 'max' but got {norm}")

    with torch.no_grad():
        acc_bin, conf_bin, prop_bin = _binning_bucketize(confidences, accuracies, bin_boundaries)

    out_dtype = confidences.dtype
    if norm == "l1":
        return torch.sum(torch.abs(acc_bin - conf_bin) * prop_bin).to(out_dtype)
    if norm == "max":
        ce = torch.max(torch.abs(acc_bin - conf_bin))
    if norm == "l2":
        ce = torch.sum(torch.pow(acc_bin - conf_bin, 2) * prop_bin)
        if debias:
            # the reference's order, (acc_bin - 1) rather than (1 - acc_bin) of Kumar et al. 2019
            debias_bins = (acc_bin * (acc_bin - 1) * prop_bin) / (prop_bin * accuracies.size()[0] - 1)
            ce += torch.sum(torch.nan_to_num(debias_bins))
        return torch.sqrt(ce).to(out_dtype) if ce > 0 else torch.tensor(0)
    return ce.to(out_dtype)


# ---------------------------------------------------------------------------------------------------------
# binary
# ---------------------------------------------------------------------------------------------------------
def _binary_calibration_error_arg_validation(
    n_bins: int,
    norm: Literal["l1", "l2", "max"] = "l1",
    ignore_index: Optional[int] = None,
) -> None:
    if not isinstance(n_bins, int) or n_bins < 1:
        raise ValueError(f"Expected argument `n_bins` to be an integer larger than 0, but got {n_bins}")
    allowed_norm = ("l1", "l2", "max")
    if norm not in allowed_norm:
        raise ValueError(f"Expected argument `norm` to be one of {allowed_norm}, but got {norm}.")
    if ignore_index is not None and not isinstance(ignore_index, int):
        raise ValueError(f"Expected argument `ignore_index` to either be `None` or an integer, but got {ignore_index}")


def _binary_calibration_error_tensor_validation(
    preds: Tensor, target: Tensor, ignore_index: Optional[int] = None
) -> None:
    """Same shape, targets in {0, 1} (+ ignore_index), floating scores (reference :143-152 with the binary confusion-matrix
    checks of confusion_matrix.py:80-116).  The content checks synchronise the host, as the reference's do."""
    _check_same_shape(preds, target)
    bad = (target != 0) & (target != 1)
    if ignore_index is not None:
        bad &= target != ignore_index
    if bool(bad.any()):
        raise RuntimeError(
            f"Detected the following values in `target`: {torch.unique(target)} but expected only"
            f" the following values {[0, 1] if ignore_index is None else [ignore_index]}."
        )
    if not preds.is_floating_point():
        if bool(((preds != 0) & (preds != 1)).any()):
            raise RuntimeError(
                f"Detected the following values in `preds`: {torch.unique(preds)} but expected only"
                " the following values [0,1] since preds is a label tensor."
            )
        raise ValueError(
            "Expected argument `preds` to be floating tensor with probabilities/logits"
            f" but got tensor with dtype {preds.dtype}"
        )


def _binary_calibration_error_format(
    preds: Tensor, target: Tensor, ignore_index: Optional[int] = None
) -> tuple[Tensor, Tensor]:
    """``_binary_confusion_matrix_format(..., convert_to_labels=False)`` (reference confusion_matrix.py:119-144): flatten,
    drop ignored samples, sigmoid if the batch holds logits (kernel K6, no host sync)."""
    preds = preds.flatten()
    target = target.flatten()
    if ignore_index is not None:
        keep = target != ignore_index
        preds, target = preds[keep], target[keep]
    if preds.is_floating_point():
        preds = _native.sigmoid_if_logits(preds)
    return preds, target


def _binary_calibration_error_update(preds: Tensor, target: Tensor) -> tuple[Tensor, Tensor]:
    confidences, accuracies = preds, target
    return confidences, accuracies


def binary_calibration_error(
    preds: Tensor,
    target: Tensor,
    n_bins: int = 15,
    norm: Literal["l1", "l2", "max"] = "l1",
    ignore_index: Optional[int] = None,
    validate_args: bool = True,
) -> Tensor:
    r"""`Top-label Calibration Error`_ for binary tasks (reference :155-228).

    ``preds``: ``(N, ...)`` float probabilities or logits (sigmoid applied when any score lies outside [0, 1]);
    ``target``: ``(N, ...)`` labels in {0, 1}.  Extra dimensions are flattened into the batch.  Inputs must be CUDA tensors.

    Example:
        >>> preds = torch.tensor([0.25, 0.25, 0.55, 0.75, 0.75], device="cuda")
        >>> target = torch.tensor([0, 0, 1, 1, 1], device="cuda")
        >>> binary_calibration_error(preds, target, n_bins=2, norm='l1')
        tensor(0.2900, device='cuda:0')

    """
    if validate_args:
        _binary_calibration_error_arg_validation(n_bins, norm, ignore_index)
        _binary_calibration_error_tensor_validation(preds, target, ignore_index)
    preds, target = _binary_calibration_error_format(preds, target, ignore_index)
    confidences, accuracies = _binary_calibration_error_update(preds, target)
    return _ce_compute(confidences, accuracies, n_bins, norm)


# ---------------------------------------------------------------------------------------------------------
# multiclass
# ---------------------------------------------------------------------------------------------------------
def _multiclass_calibration_error_arg_validation(
    num_classes: int,
    n_bins: int,
    norm: Literal["l1", "l2", "max"] = "l1",
    ignore_index: Optional[int] = None,
) -> None:
    if not isinstance(num_classes, int) or num_classes < 2:
        raise ValueError(f"Expected argument `num_classes` to be an integer larger than 1, but got {num_classes}")
    if not isinstance(n_bins, int) or n_bins < 1:
        raise ValueError(f"Expected argument `n_bins` to be an integer larger than 0, but got {n_bins}")
    allowed_norm = ("l1", "l2", "max")
    if norm not in allowed_norm:
        raise ValueError(f"Expected argument `norm` to be one of {allowed_norm}, but got {norm}.")
    if ignore_index is not None and not isinstance(ignore_index, int):
        raise ValueError(f"Expected argument `ignore_index` to either be `None` or an integer, but got {ignore_index}")


def _multiclass_calibration_error_tensor_validation(
    preds: Tensor, target: Tensor, num_classes: int, ignore_index: Optional[int] = None
) -> None:
    """Shape rules and floating scores (reference :231-236).  Target *values* are range-checked inside kernel K14a."""
    check_multiclass_shapes(preds, target, num_classes)
    if not preds.is_floating_point():
        raise ValueError(
            "Expected argument `preds` to be floating tensor with probabilities/logits"
            f" but got tensor with dtype {preds.dtype}"
        )


def _rows(preds: Tensor) -> Tensor:
    """``[N, C, d...]`` -> ``[N * d..., C]`` (``movedim(1, -1)``; a copy only when there are trailing dims)."""
    if preds.ndim == 2:
        return preds
    return torch.movedim(preds, 1, -1).reshape(-1, preds.shape[1])


def _multiclass_calibration_error_update(
    preds: Tensor,
    target: Tensor,
) -> tuple[Tensor, Tensor]:
    """``normalize_logits_if_needed(preds, "softmax").max(dim=1)`` and ``argmax == target`` of formatted ``[M, C]`` rows
    (reference :239-246), one kernel (K14a).  Returns float32 ``(confidences, accuracies)``."""
    return _native.calibration_top_label(preds, target)


def _multiclass_calibration_error_fused_update(
    preds: Tensor, target: Tensor, num_classes: int, ignore_index: Optional[int] = None, validate_args: bool = False
) -> tuple[Tensor, Tensor]:
    """Format + update in one pass over the scores: ignored rows are left out of the logits vote inside K14a and dropped
    from its ``[N]`` outputs afterwards (one host sync, as the reference's boolean index; none without ``ignore_index``).
    ``validate_args``: the kernel range-checks every kept target; the error word is read back before anything is
    returned."""
    preds = _rows(preds)
    target = target.flatten()
    flag = new_flag(preds.device) if validate_args else None
    confidences, accuracies = _native.calibration_top_label(preds, target, ignore_index, flag)
    if flag is not None:
        raise_if_flagged(flag, num_classes, ignore_index)
    if ignore_index is not None:
        keep = target != ignore_index
        confidences, accuracies = confidences[keep], accuracies[keep]
    return confidences, accuracies


def multiclass_calibration_error(
    preds: Tensor,
    target: Tensor,
    num_classes: int,
    n_bins: int = 15,
    norm: Literal["l1", "l2", "max"] = "l1",
    ignore_index: Optional[int] = None,
    validate_args: bool = True,
) -> Tensor:
    r"""`Top-label Calibration Error`_ for multiclass tasks (reference :249-323).

    ``preds``: ``(N, C, ...)`` float probabilities or logits (row softmax applied when any kept score lies outside
    [0, 1]); ``target``: ``(N, ...)`` labels.  Extra dimensions are flattened into the batch.  Inputs must be CUDA tensors.

    Example:
        >>> preds = torch.tensor([[0.25, 0.20, 0.55], [0.55, 0.05, 0.40], [0.10, 0.30, 0.60], [0.90, 0.05, 0.05]],
        ...                      device="cuda")
        >>> target = torch.tensor([0, 1, 2, 0], device="cuda")
        >>> multiclass_calibration_error(preds, target, num_classes=3, n_bins=3, norm='l1')
        tensor(0.2000, device='cuda:0')

    """
    if validate_args:
        _multiclass_calibration_error_arg_validation(num_classes, n_bins, norm, ignore_index)
        _multiclass_calibration_error_tensor_validation(preds, target, num_classes, ignore_index)
    confidences, accuracies = _multiclass_calibration_error_fused_update(preds, target, num_classes, ignore_index, validate_args)
    return _ce_compute(confidences, accuracies, n_bins, norm)


def calibration_error(
    preds: Tensor,
    target: Tensor,
    task: Literal["binary", "multiclass"],
    n_bins: int = 15,
    norm: Literal["l1", "l2", "max"] = "l1",
    num_classes: Optional[int] = None,
    ignore_index: Optional[int] = None,
    validate_args: bool = True,
) -> Tensor:
    r"""`Top-label Calibration Error`_: dispatches to :func:`binary_calibration_error` or
    :func:`multiclass_calibration_error` by ``task`` (reference :326-372)."""
    task = ClassificationTaskNoMultilabel.from_str(task)
    assert norm is not None  # noqa: S101
    if task == ClassificationTaskNoMultilabel.BINARY:
        return binary_calibration_error(preds, target, n_bins, norm, ignore_index, validate_args)
    if task == ClassificationTaskNoMultilabel.MULTICLASS:
        if not isinstance(num_classes, int):
            raise ValueError(f"`num_classes` is expected to be `int` but `{type(num_classes)} was passed.`")
        return multiclass_calibration_error(preds, target, num_classes, n_bins, norm, ignore_index, validate_args)
    raise ValueError(f"Expected argument `task` to either be `'binary'` or `'multiclass'` but got {task}")
