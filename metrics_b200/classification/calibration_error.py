"""Top-label calibration error, modular (reference: classification/calibration_error.py).

``update`` appends this batch's confidences and accuracies to the ``cat`` states (binary: the formatted scores and targets;
multiclass: kernel K14a, one read of the ``[N, C]`` scores); ``compute`` bins them with kernel K14b and applies the
reference's epilogue (functional/classification/calibration_error.py)."""
from typing import Any, List, Optional

from torch import Tensor
from typing_extensions import Literal

from metrics_b200.classification.base import _ClassificationTaskWrapper
from metrics_b200.functional.classification.calibration_error import (
    _binary_calibration_error_arg_validation,
    _binary_calibration_error_format,
    _binary_calibration_error_tensor_validation,
    _binary_calibration_error_update,
    _ce_compute,
    _multiclass_calibration_error_arg_validation,
    _multiclass_calibration_error_fused_update,
    _multiclass_calibration_error_tensor_validation,
)
from metrics_b200.metric import Metric
from metrics_b200.utilities.data import dim_zero_cat
from metrics_b200.utilities.enums import ClassificationTaskNoMultilabel


class BinaryCalibrationError(Metric):
    r"""`Top-label Calibration Error`_ for binary tasks (reference :36-157).

    ``preds``: ``(N, ...)`` float probabilities or logits; ``target``: ``(N, ...)`` labels in {0, 1}.  ``compute`` returns
    the l1 (ECE), l2 (RMSCE) or max (MCE) calibration error over ``n_bins`` uniform bins of [0, 1]."""

    is_differentiable: bool = False
    higher_is_better: bool = False
    full_state_update: bool = False
    plot_lower_bound: float = 0.0
    plot_upper_bound: float = 1.0

    confidences: List[Tensor]
    accuracies: List[Tensor]

    def __init__(
        self,
        n_bins: int = 15,
        norm: Literal["l1", "l2", "max"] = "l1",
        ignore_index: Optional[int] = None,
        validate_args: bool = True,
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        if validate_args:
            _binary_calibration_error_arg_validation(n_bins, norm, ignore_index)
        self.validate_args = validate_args
        self.n_bins = n_bins
        self.norm = norm
        self.ignore_index = ignore_index
        self.add_state("confidences", [], dist_reduce_fx="cat")
        self.add_state("accuracies", [], dist_reduce_fx="cat")

    def update(self, preds: Tensor, target: Tensor) -> None:
        """Update metric states with predictions and targets."""
        if self.validate_args:
            _binary_calibration_error_tensor_validation(preds, target, self.ignore_index)
        preds, target = _binary_calibration_error_format(preds, target, self.ignore_index)
        confidences, accuracies = _binary_calibration_error_update(preds, target)
        self.confidences.append(confidences)
        self.accuracies.append(accuracies)

    def compute(self) -> Tensor:
        """Compute metric."""
        confidences = dim_zero_cat(self.confidences)
        accuracies = dim_zero_cat(self.accuracies)
        return _ce_compute(confidences, accuracies, self.n_bins, norm=self.norm)


class MulticlassCalibrationError(Metric):
    r"""`Top-label Calibration Error`_ for multiclass tasks (reference :160-294).

    ``preds``: ``(N, C, ...)`` float probabilities or logits; ``target``: ``(N, ...)`` labels.  The states hold one float32
    confidence (the top softmax probability) and one float32 accuracy (top label == target) per kept sample."""

    is_differentiable: bool = False
    higher_is_better: bool = False
    full_state_update: bool = False
    plot_lower_bound: float = 0.0
    plot_upper_bound: float = 1.0
    plot_legend_name: str = "Class"

    confidences: List[Tensor]
    accuracies: List[Tensor]

    def __init__(
        self,
        num_classes: int,
        n_bins: int = 15,
        norm: Literal["l1", "l2", "max"] = "l1",
        ignore_index: Optional[int] = None,
        validate_args: bool = True,
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        if validate_args:
            _multiclass_calibration_error_arg_validation(num_classes, n_bins, norm, ignore_index)
        self.validate_args = validate_args
        self.num_classes = num_classes
        self.n_bins = n_bins
        self.norm = norm
        self.ignore_index = ignore_index
        self.add_state("confidences", [], dist_reduce_fx="cat")
        self.add_state("accuracies", [], dist_reduce_fx="cat")

    def update(self, preds: Tensor, target: Tensor) -> None:
        """Update metric states with predictions and targets."""
        if self.validate_args:
            _multiclass_calibration_error_tensor_validation(preds, target, self.num_classes, self.ignore_index)
        confidences, accuracies = _multiclass_calibration_error_fused_update(
            preds, target, self.num_classes, self.ignore_index, self.validate_args
        )
        self.confidences.append(confidences)
        self.accuracies.append(accuracies)

    def compute(self) -> Tensor:
        """Compute metric."""
        confidences = dim_zero_cat(self.confidences)
        accuracies = dim_zero_cat(self.accuracies)
        return _ce_compute(confidences, accuracies, self.n_bins, norm=self.norm)


class CalibrationError(_ClassificationTaskWrapper):
    r"""`Top-label Calibration Error`_: ``CalibrationError(task="binary" | "multiclass", ...)`` returns a
    :class:`BinaryCalibrationError` or a :class:`MulticlassCalibrationError` (reference :297-352)."""

    def __new__(  # type: ignore[misc]
        cls: type["CalibrationError"],
        task: Literal["binary", "multiclass"],
        n_bins: int = 15,
        norm: Literal["l1", "l2", "max"] = "l1",
        num_classes: Optional[int] = None,
        ignore_index: Optional[int] = None,
        validate_args: bool = True,
        **kwargs: Any,
    ) -> Metric:
        """Initialize task metric."""
        task = ClassificationTaskNoMultilabel.from_str(task)
        kwargs.update({"n_bins": n_bins, "norm": norm, "ignore_index": ignore_index, "validate_args": validate_args})
        if task == ClassificationTaskNoMultilabel.BINARY:
            return BinaryCalibrationError(**kwargs)
        if task == ClassificationTaskNoMultilabel.MULTICLASS:
            if not isinstance(num_classes, int):
                raise ValueError(f"`num_classes` is expected to be `int` but `{type(num_classes)} was passed.`")
            return MulticlassCalibrationError(num_classes, **kwargs)
        raise ValueError(f"Not handled value: {task}")
