"""The retrieval metric classes (reference: src/torchmetrics/retrieval/*.py).  Each one names its K16 metric kind and the
arguments of that kind; the grouping, empty-query handling and aggregation are in `RetrievalMetric`."""
from typing import Any, Callable, Optional, Union

from torch import Tensor
from typing_extensions import Literal

from metrics_b200 import _native
from metrics_b200.functional.retrieval import (
    retrieval_average_precision,
    retrieval_fall_out,
    retrieval_hit_rate,
    retrieval_normalized_dcg,
    retrieval_precision,
    retrieval_r_precision,
    retrieval_recall,
    retrieval_reciprocal_rank,
)
from metrics_b200.functional.retrieval._metrics import _FLOAT_R_MESSAGE
from metrics_b200.retrieval.base import RetrievalMetric


def _check_top_k(top_k: Optional[int]) -> None:
    if top_k is not None and not (isinstance(top_k, int) and top_k > 0):
        raise ValueError("`top_k` has to be a positive integer or None")


class RetrievalMAP(RetrievalMetric):
    """Mean average precision over the queries (reference retrieval/average_precision.py)."""

    is_differentiable: bool = False
    higher_is_better: bool = True
    full_state_update: bool = False
    _kind = _native.RET_AP

    def __init__(
        self,
        empty_target_action: str = "neg",
        ignore_index: Optional[int] = None,
        top_k: Optional[int] = None,
        aggregation: Union[Literal["mean", "median", "min", "max"], Callable] = "mean",
        **kwargs: Any,
    ) -> None:
        super().__init__(empty_target_action=empty_target_action, ignore_index=ignore_index, aggregation=aggregation, **kwargs)
        if top_k is not None and not isinstance(top_k, int) and top_k <= 0:
            raise ValueError(f"Argument ``top_k`` has to be a positive integer or None, but got {top_k}")
        self.k = top_k

    def _metric_args(self) -> dict:
        return {"top_k": self.k}

    def _metric(self, preds: Tensor, target: Tensor) -> Tensor:
        return retrieval_average_precision(preds, target, top_k=self.k)


class RetrievalMRR(RetrievalMetric):
    """Mean reciprocal rank over the queries (reference retrieval/reciprocal_rank.py)."""

    is_differentiable: bool = False
    higher_is_better: bool = True
    full_state_update: bool = False
    _kind = _native.RET_RR

    def __init__(
        self,
        empty_target_action: str = "neg",
        ignore_index: Optional[int] = None,
        top_k: Optional[int] = None,
        aggregation: Union[Literal["mean", "median", "min", "max"], Callable] = "mean",
        **kwargs: Any,
    ) -> None:
        super().__init__(empty_target_action=empty_target_action, ignore_index=ignore_index, aggregation=aggregation, **kwargs)
        if top_k is not None and not isinstance(top_k, int) and top_k <= 0:
            raise ValueError(f"Argument ``top_k`` has to be a positive integer or None, but got {top_k}")
        self.top_k = top_k

    def _metric_args(self) -> dict:
        return {"top_k": self.top_k}

    def _metric(self, preds: Tensor, target: Tensor) -> Tensor:
        return retrieval_reciprocal_rank(preds, target, top_k=self.top_k)


class RetrievalPrecision(RetrievalMetric):
    """Precision at ``top_k`` over the queries (reference retrieval/precision.py)."""

    is_differentiable: bool = False
    higher_is_better: bool = True
    full_state_update: bool = False
    _kind = _native.RET_PRECISION

    def __init__(
        self,
        empty_target_action: str = "neg",
        ignore_index: Optional[int] = None,
        top_k: Optional[int] = None,
        adaptive_k: bool = False,
        aggregation: Union[Literal["mean", "median", "min", "max"], Callable] = "mean",
        **kwargs: Any,
    ) -> None:
        super().__init__(empty_target_action=empty_target_action, ignore_index=ignore_index, aggregation=aggregation, **kwargs)
        _check_top_k(top_k)
        if not isinstance(adaptive_k, bool):
            raise ValueError("`adaptive_k` has to be a boolean")
        self.top_k = top_k
        self.adaptive_k = adaptive_k

    def _metric_args(self) -> dict:
        return {"top_k": self.top_k, "adaptive_k": self.adaptive_k}

    def _metric(self, preds: Tensor, target: Tensor) -> Tensor:
        return retrieval_precision(preds, target, top_k=self.top_k, adaptive_k=self.adaptive_k)


class RetrievalRecall(RetrievalMetric):
    """Recall at ``top_k`` over the queries (reference retrieval/recall.py)."""

    is_differentiable: bool = False
    higher_is_better: bool = True
    full_state_update: bool = False
    _kind = _native.RET_RECALL

    def __init__(
        self,
        empty_target_action: str = "neg",
        ignore_index: Optional[int] = None,
        top_k: Optional[int] = None,
        aggregation: Union[Literal["mean", "median", "min", "max"], Callable] = "mean",
        **kwargs: Any,
    ) -> None:
        super().__init__(empty_target_action=empty_target_action, ignore_index=ignore_index, aggregation=aggregation, **kwargs)
        _check_top_k(top_k)
        self.top_k = top_k

    def _metric_args(self) -> dict:
        return {"top_k": self.top_k}

    def _metric(self, preds: Tensor, target: Tensor) -> Tensor:
        return retrieval_recall(preds, target, top_k=self.top_k)


class RetrievalHitRate(RetrievalMetric):
    """Hit rate at ``top_k`` over the queries (reference retrieval/hit_rate.py)."""

    is_differentiable: bool = False
    higher_is_better: bool = True
    full_state_update: bool = False
    _kind = _native.RET_HIT_RATE

    def __init__(
        self,
        empty_target_action: str = "neg",
        ignore_index: Optional[int] = None,
        top_k: Optional[int] = None,
        aggregation: Union[Literal["mean", "median", "min", "max"], Callable] = "mean",
        **kwargs: Any,
    ) -> None:
        super().__init__(empty_target_action=empty_target_action, ignore_index=ignore_index, aggregation=aggregation, **kwargs)
        _check_top_k(top_k)
        self.top_k = top_k

    def _metric_args(self) -> dict:
        return {"top_k": self.top_k}

    def _metric(self, preds: Tensor, target: Tensor) -> Tensor:
        return retrieval_hit_rate(preds, target, top_k=self.top_k)


class RetrievalFallOut(RetrievalMetric):
    """Fall-out at ``top_k`` over the queries (reference retrieval/fall_out.py).  A query is empty when it has no negative
    target; the default action counts it as 1."""

    is_differentiable: bool = False
    higher_is_better: bool = False
    full_state_update: bool = False
    _kind = _native.RET_FALL_OUT
    _empty_message = "`compute` method was provided with a query with no negative target."

    def __init__(
        self,
        empty_target_action: str = "pos",
        ignore_index: Optional[int] = None,
        top_k: Optional[int] = None,
        aggregation: Union[Literal["mean", "median", "min", "max"], Callable] = "mean",
        **kwargs: Any,
    ) -> None:
        super().__init__(empty_target_action=empty_target_action, ignore_index=ignore_index, aggregation=aggregation, **kwargs)
        _check_top_k(top_k)
        self.top_k = top_k

    def _metric_args(self) -> dict:
        return {"top_k": self.top_k}

    def _metric(self, preds: Tensor, target: Tensor) -> Tensor:
        return retrieval_fall_out(preds, target, top_k=self.top_k)


class RetrievalRPrecision(RetrievalMetric):
    """R-precision over the queries (reference retrieval/r_precision.py)."""

    is_differentiable: bool = False
    higher_is_better: bool = True
    full_state_update: bool = False
    _kind = _native.RET_R_PRECISION

    def compute(self) -> Tensor:
        """Per-query R-precision; like the reference, float targets in a non-empty query raise ``TypeError``."""
        if any(t.is_floating_point() for t in self.target) and not bool(self._empty_flags().all()):
            raise TypeError(_FLOAT_R_MESSAGE)
        return super().compute()

    def _metric(self, preds: Tensor, target: Tensor) -> Tensor:
        return retrieval_r_precision(preds, target)


class RetrievalNormalizedDCG(RetrievalMetric):
    """Normalized DCG at ``top_k`` over the queries, graded targets allowed (reference retrieval/ndcg.py)."""

    is_differentiable: bool = False
    higher_is_better: bool = True
    full_state_update: bool = False
    _kind = _native.RET_NDCG

    def __init__(
        self,
        empty_target_action: str = "neg",
        ignore_index: Optional[int] = None,
        top_k: Optional[int] = None,
        aggregation: Union[Literal["mean", "median", "min", "max"], Callable] = "mean",
        **kwargs: Any,
    ) -> None:
        super().__init__(empty_target_action=empty_target_action, ignore_index=ignore_index, aggregation=aggregation, **kwargs)
        _check_top_k(top_k)
        self.top_k = top_k
        self.allow_non_binary_target = True

    def _metric_args(self) -> dict:
        return {"top_k": self.top_k}

    def _metric(self, preds: Tensor, target: Tensor) -> Tensor:
        return retrieval_normalized_dcg(preds, target, top_k=self.top_k)
