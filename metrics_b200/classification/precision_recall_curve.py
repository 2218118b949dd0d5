"""Precision-recall-curve metric classes, exact mode (reference: classification/precision_recall_curve.py).

States are the reference's: list states ``preds`` / ``target`` with ``dist_reduce_fx="cat"`` (observable through
``metric_state``, compute groups, ``state_dict``).  ``update`` runs the format kernel (conditional sigmoid/softmax) and
appends; ``compute`` concatenates once and runs the batched sort + scan pipeline.
"""
from __future__ import annotations

from typing import Any, List, Optional, Union

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200.functional.classification.precision_recall_curve import (
    _adjust_threshold_arg,
    _binary_precision_recall_curve_arg_validation,
    _binary_precision_recall_curve_compute,
    _binary_precision_recall_curve_format,
    _binary_precision_recall_curve_tensor_validation,
    _binary_precision_recall_curve_update,
    _multiclass_precision_recall_curve_arg_validation,
    _multiclass_precision_recall_curve_compute,
    _multiclass_precision_recall_curve_format,
    _multiclass_precision_recall_curve_tensor_validation,
    _multiclass_precision_recall_curve_update,
    _multilabel_precision_recall_curve_arg_validation,
    _multilabel_precision_recall_curve_compute,
    _multilabel_precision_recall_curve_format,
    _multilabel_precision_recall_curve_tensor_validation,
    _multilabel_precision_recall_curve_update,
)
from metrics_b200.metric import Metric
from metrics_b200.utilities.data import dim_zero_cat


class BinaryPrecisionRecallCurve(Metric):
    """Reference :55-177."""

    is_differentiable: bool = False
    higher_is_better: Optional[bool] = None
    full_state_update: bool = False

    def __init__(
        self,
        thresholds: Optional[Union[int, List[float], Tensor]] = None,
        ignore_index: Optional[int] = None,
        validate_args: bool = True,
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        if validate_args:
            _binary_precision_recall_curve_arg_validation(thresholds, ignore_index)
        self.ignore_index = ignore_index
        self.validate_args = validate_args
        self._install_curve_states(thresholds, lambda n_thr: (n_thr, 2, 2))

    def _install_curve_states(self, thresholds, binned_shape) -> None:
        """Exact mode (``thresholds=None``): list states ``preds`` / ``target`` (``cat``).  Binned mode: a non-persistent
        ``thresholds`` buffer and ONE constant-size int64 ``confmat`` state of shape ``binned_shape(T)`` (``sum``)."""
        grid = _adjust_threshold_arg(thresholds)
        if grid is None:
            self.thresholds = None
            for name in ("preds", "target"):
                self.add_state(name, default=[], dist_reduce_fx="cat")
        else:
            self.register_buffer("thresholds", grid, persistent=False)
            self.add_state("confmat", default=torch.zeros(*binned_shape(len(grid)), dtype=torch.long), dist_reduce_fx="sum")
        # One sort + scan yields AUROC *and* AP: members of a MetricCollection compute group share this dict by reference
        # (collections.py links it like a state), so the second metric of the group reuses the first one's evaluation.
        self._group_cache: dict = {}

    def _accumulate(self, state) -> None:
        """Fold one batch's functional state into the metric: add the binned counts, or keep the formatted batch."""
        if isinstance(state, Tensor):
            self.confmat += state
        else:
            self.preds.append(state[0])
            self.target.append(state[1])

    def reset(self) -> None:
        self._group_cache.clear()
        Metric.reset(self)

    def _cache_put(self, key, value) -> None:
        if len(self._group_cache) >= 4:  # synced states get a fresh identity per sync(): do not accumulate stale entries
            self._group_cache.clear()
        self._group_cache[key] = value

    def _curve_scalars(self, num_classes: int = 1, pos_label: int = 1):
        """``(auroc, ap, counts)`` of the current state from ONE `mb200_curve_evaluate` call, memoised until the next
        update / reset.  Keyed by the identity of the state object, so synced states never hit a local entry."""
        from metrics_b200 import _native

        if self.thresholds is not None:
            return None  # binned mode: the compute functions work on the confmat state
        key = (id(self.preds), id(self.target), num_classes, pos_label, bool(getattr(self, "_sharded_now", False)))
        hit = self._group_cache.get(key)
        if getattr(self, "_sharded_now", False):
            from metrics_b200.parallel_curves import ovr_curve_scalars_sharded

            has = len(self.preds) > 0 if isinstance(self.preds, list) else self.preds.numel() > 0
            preds, target = self._state() if has else (None, None)
            hit = ovr_curve_scalars_sharded(preds, target, num_classes, self.process_group, self.device, cached=hit)
            self._cache_put(key, hit)
            return hit
        if hit is None:
            preds, target = self._state()
            if preds.numel() == 0:
                raise IndexError("metrics_b200: cannot evaluate a curve metric without samples")
            auroc, ap, counts, _ = _native.curve_evaluate(preds, target, num_classes, pos_label, want_curve=False,
                                                          unit_range=True)  # states are post-format
            hit = (auroc, ap, counts)
            self._cache_put(key, hit)
        return hit

    def update(self, preds: Tensor, target: Tensor) -> None:
        self._group_cache.clear()
        if self.validate_args:
            _binary_precision_recall_curve_tensor_validation(preds, target, self.ignore_index)
        preds, target, _ = _binary_precision_recall_curve_format(preds, target, self.thresholds, self.ignore_index)
        state = _binary_precision_recall_curve_update(preds, target, self.thresholds)
        self._accumulate(state)

    def _state(self):
        if self.thresholds is not None:
            return self.confmat
        return dim_zero_cat(self.preds), dim_zero_cat(self.target)

    def compute(self) -> tuple[Tensor, Tensor, Tensor]:
        return _binary_precision_recall_curve_compute(self._state(), self.thresholds)


class MulticlassPrecisionRecallCurve(Metric):
    """Reference :228-380."""

    is_differentiable: bool = False
    higher_is_better: Optional[bool] = None
    full_state_update: bool = False

    def __init__(
        self,
        num_classes: int,
        thresholds: Optional[Union[int, List[float], Tensor]] = None,
        average: Optional[Literal["micro", "macro"]] = None,
        ignore_index: Optional[int] = None,
        validate_args: bool = True,
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        if validate_args:
            _multiclass_precision_recall_curve_arg_validation(num_classes, thresholds, ignore_index, average)
        self.num_classes = num_classes
        self.average = average
        self.ignore_index = ignore_index
        self.validate_args = validate_args
        # binned mode (reference :353-359): micro average keeps the binary [T, 2, 2] layout
        self._install_curve_states(thresholds, lambda n_thr: (n_thr, 2, 2) if average == "micro" else (n_thr, num_classes, 2, 2))

    reset = BinaryPrecisionRecallCurve.reset
    _curve_scalars = BinaryPrecisionRecallCurve._curve_scalars
    _cache_put = BinaryPrecisionRecallCurve._cache_put
    _install_curve_states = BinaryPrecisionRecallCurve._install_curve_states
    _accumulate = BinaryPrecisionRecallCurve._accumulate

    def update(self, preds: Tensor, target: Tensor) -> None:
        self._group_cache.clear()
        if self.validate_args:
            _multiclass_precision_recall_curve_tensor_validation(preds, target, self.num_classes, self.ignore_index)
        preds, target, _ = _multiclass_precision_recall_curve_format(
            preds, target, self.num_classes, self.thresholds, self.ignore_index, self.average
        )
        state = _multiclass_precision_recall_curve_update(preds, target, self.num_classes, self.thresholds, self.average)
        self._accumulate(state)

    _state = BinaryPrecisionRecallCurve._state

    def compute(self):
        return _multiclass_precision_recall_curve_compute(self._state(), self.num_classes, self.thresholds, self.average)


class MultilabelPrecisionRecallCurve(Metric):
    """Reference :383-597.  States: ``preds`` / ``target`` lists of ``[N, L]`` batches (exact) or the ``[T, L, 2, 2]``
    multi-threshold confusion matrix (binned)."""

    is_differentiable: bool = False
    higher_is_better: Optional[bool] = None
    full_state_update: bool = False

    def __init__(
        self,
        num_labels: int,
        thresholds: Optional[Union[int, List[float], Tensor]] = None,
        ignore_index: Optional[int] = None,
        validate_args: bool = True,
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        if validate_args:
            _multilabel_precision_recall_curve_arg_validation(num_labels, thresholds, ignore_index)
        self.num_labels = num_labels
        self.ignore_index = ignore_index
        self.validate_args = validate_args
        self._install_curve_states(thresholds, lambda n_thr: (n_thr, num_labels, 2, 2))

    reset = BinaryPrecisionRecallCurve.reset
    _cache_put = BinaryPrecisionRecallCurve._cache_put
    _state = BinaryPrecisionRecallCurve._state
    _install_curve_states = BinaryPrecisionRecallCurve._install_curve_states
    _accumulate = BinaryPrecisionRecallCurve._accumulate

    def _curve_scalars(self):
        """Per-label ``(auroc, ap, counts)`` from ONE `mb200_curve_evaluate_multilabel` call, shared by the members of a
        compute group (see BinaryPrecisionRecallCurve._curve_scalars)."""
        from metrics_b200 import _native

        if self.thresholds is not None:
            return None
        key = (id(self.preds), id(self.target), "multilabel", self.num_labels, self.ignore_index)
        hit = self._group_cache.get(key)
        if hit is None:
            preds, target = self._state()
            if preds.numel() == 0:
                raise IndexError("metrics_b200: cannot evaluate a curve metric without samples")
            auroc, ap, counts, _ = _native.curve_evaluate_multilabel(preds, target, self.num_labels, self.ignore_index)
            hit = (auroc, ap, counts)
            self._cache_put(key, hit)
        return hit

    def update(self, preds: Tensor, target: Tensor) -> None:
        self._group_cache.clear()
        if self.validate_args:
            _multilabel_precision_recall_curve_tensor_validation(preds, target, self.num_labels, self.ignore_index)
        preds, target, _ = _multilabel_precision_recall_curve_format(
            preds, target, self.num_labels, self.thresholds, self.ignore_index
        )
        state = _multilabel_precision_recall_curve_update(preds, target, self.num_labels, self.thresholds, self.ignore_index)
        self._accumulate(state)

    def compute(self):
        return _multilabel_precision_recall_curve_compute(self._state(), self.num_labels, self.thresholds, self.ignore_index)


from metrics_b200.classification.base import _ClassificationTaskWrapper  # noqa: E402
from metrics_b200.classification._curve_common import build_for_task  # noqa: E402


class PrecisionRecallCurve(_ClassificationTaskWrapper):
    """Task wrapper (reference :600-692)."""

    def __new__(  # type: ignore[misc]
        cls,
        task: Literal["binary", "multiclass", "multilabel"],
        thresholds: Optional[Union[int, List[float], Tensor]] = None,
        num_classes: Optional[int] = None,
        num_labels: Optional[int] = None,
        ignore_index: Optional[int] = None,
        validate_args: bool = True,
        **kwargs: Any,
    ) -> Metric:
        shared = dict(kwargs, thresholds=thresholds, ignore_index=ignore_index, validate_args=validate_args)
        return build_for_task(task, num_classes, num_labels, lambda: BinaryPrecisionRecallCurve(**shared),
                              lambda c: MulticlassPrecisionRecallCurve(c, **shared),
                              lambda n: MultilabelPrecisionRecallCurve(n, **shared))
