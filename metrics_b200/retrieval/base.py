"""Base class of the retrieval metrics (reference: retrieval/base.py).  ``update`` keeps the reference's validation and
its three list states; ``compute`` groups the records by query on the GPU (kernel K16: one group sort, then one evaluation
launch per metric) instead of a Python loop over the queries."""
from abc import ABC, abstractmethod
from typing import Any, Callable, List, Optional, Union

import torch
from torch import Tensor, tensor
from typing_extensions import Literal

from metrics_b200 import _native
from metrics_b200.metric import Metric
from metrics_b200.utilities.checks import _check_retrieval_inputs
from metrics_b200.utilities.data import dim_zero_cat


def _retrieval_aggregate(
    values: Tensor,
    aggregation: Union[Literal["mean", "median", "min", "max"], Callable] = "mean",
    dim: Optional[int] = None,
) -> Tensor:
    """Aggregate the per-query values into one value (reference base.py:26-40)."""
    if aggregation == "mean":
        return values.mean() if dim is None else values.mean(dim=dim)
    if aggregation == "median":
        return values.median() if dim is None else values.median(dim=dim).values
    if aggregation == "min":
        return values.min() if dim is None else values.min(dim=dim).values
    if aggregation == "max":
        return values.max() if dim is None else values.max(dim=dim).values
    return aggregation(values, dim=dim)


class RetrievalMetric(Metric, ABC):
    """Retrieval metric over queries identified by ``indexes`` (reference base.py:43-191).

    ``update(preds, target, indexes)`` checks and flattens the batch and appends it to the list states ``indexes``,
    ``preds`` (float32) and ``target`` (int64, or float32 for floating targets).  ``compute`` evaluates every query, in
    ascending index order, with ``empty_target_action`` for queries without a positive target (``'neg'``: 0, ``'pos'``:
    1, ``'skip'``: left out, 0 when all are, ``'error'``: ``ValueError``) and reduces the float32 values with
    ``aggregation``.  Within a query, documents are ranked by descending score; equal scores keep their order of arrival.
    The group sort is shared by every metric of a compute group (``_group_cache``)."""

    is_differentiable: bool = False
    higher_is_better: bool = True
    full_state_update: bool = False

    indexes: List[Tensor]
    preds: List[Tensor]
    target: List[Tensor]

    _kind: int = -1
    _empty_message = "`compute` method was provided with a query with no positive target."

    def __init__(
        self,
        empty_target_action: str = "neg",
        ignore_index: Optional[int] = None,
        aggregation: Union[Literal["mean", "median", "min", "max"], Callable] = "mean",
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        self.allow_non_binary_target = False

        empty_target_action_options = ("error", "skip", "neg", "pos")
        if empty_target_action not in empty_target_action_options:
            raise ValueError(f"Argument `empty_target_action` received a wrong value `{empty_target_action}`.")
        self.empty_target_action = empty_target_action

        if ignore_index is not None and not isinstance(ignore_index, int):
            raise ValueError("Argument `ignore_index` must be an integer or None.")
        self.ignore_index = ignore_index

        if not (aggregation in ("mean", "median", "min", "max") or callable(aggregation)):
            raise ValueError(
                "Argument `aggregation` must be one of `mean`, `median`, `min`, `max` or a custom callable function"
                f"which takes tensor of values, but got {aggregation}."
            )
        self.aggregation = aggregation

        self.add_state("indexes", default=[], dist_reduce_fx=None)
        self.add_state("preds", default=[], dist_reduce_fx=None)
        self.add_state("target", default=[], dist_reduce_fx=None)
        # sorted groups of the current states, shared with the other members of a MetricCollection compute group
        self._group_cache: dict = {}

    def update(self, preds: Tensor, target: Tensor, indexes: Tensor) -> None:
        """Check shape, check and convert dtypes, flatten and add to accumulators."""
        if indexes is None:
            raise ValueError("Argument `indexes` cannot be None")
        indexes, preds, target = _check_retrieval_inputs(
            indexes, preds, target, allow_non_binary_target=self.allow_non_binary_target, ignore_index=self.ignore_index
        )
        self._group_cache.clear()
        self.indexes.append(indexes)
        self.preds.append(preds)
        self.target.append(target)

    def reset(self) -> None:
        self._group_cache.clear()
        super().reset()

    def _cached(self, what: str, make: Callable):
        key = (what, *((id(s), len(s)) if isinstance(s, list) else (id(s), -1) for s in (self.indexes, self.preds, self.target)))
        hit = self._group_cache.get(key)
        if hit is None:
            if len(self._group_cache) >= 4:  # synced states get a fresh identity per sync(): drop stale entries
                self._group_cache.clear()
            hit = make()
            self._group_cache[key] = hit
        return hit

    def _groups(self) -> "_native.RetrievalGroups":
        def make():
            indexes = dim_zero_cat(self.indexes)
            preds = dim_zero_cat(self.preds)
            target = dim_zero_cat(self.target)
            return _native.retrieval_sort(indexes, preds, target)

        return self._cached("sort", make)

    def _metric_args(self) -> dict:
        return {}

    def _empty_flags(self) -> Tensor:
        return _native.retrieval_evaluate(self._groups(), self._kind)[1]

    def _evaluate(self, groups: "_native.RetrievalGroups") -> "tuple[Tensor, Tensor]":
        """``(value float32 [Q], empty bool [Q])`` of every query from the sorted groups: one evaluation launch."""
        ideal = None
        if self._kind == _native.RET_NDCG:
            ideal = self._cached("ideal", lambda: _native.retrieval_sort_ideal(groups))
        return _native.retrieval_evaluate(groups, self._kind, ideal=ideal, **self._metric_args())

    def compute(self) -> Tensor:
        """Per-query values from one evaluation launch over the shared group sort, then empty handling and aggregation."""
        preds = dim_zero_cat(self.preds)
        value, empty = self._evaluate(self._groups())
        action = self.empty_target_action
        if action == "error":
            if bool(empty.any()):
                raise ValueError(self._empty_message)
        elif action == "skip":
            value = value[~empty]
        else:
            value = torch.where(empty, torch.ones_like(value) if action == "pos" else torch.zeros_like(value), value)
        if value.numel():
            return _retrieval_aggregate(value.to(preds), self.aggregation)
        return tensor(0.0).to(preds)

    @abstractmethod
    def _metric(self, preds: Tensor, target: Tensor) -> Tensor:
        """The metric of one query (the functional), as in the reference; ``compute`` does not call it."""
