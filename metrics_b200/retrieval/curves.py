"""RetrievalAUROC, RetrievalPrecisionRecallCurve and RetrievalRecallAtFixedPrecision (reference: retrieval/auroc.py and
retrieval/precision_recall_curve.py).  All three subclass `RetrievalMetric`, so they share its states, its update and the
group sort of a compute group: AUROC evaluates every query in one K16e launch, the curve classes in one K16f launch."""
from typing import Any, Callable, Optional, Union

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200 import _native
from metrics_b200.functional.retrieval._curves import _check_max_fpr, retrieval_auroc, retrieval_precision_recall_curve
from metrics_b200.retrieval.base import RetrievalMetric, _retrieval_aggregate
from metrics_b200.utilities.data import dim_zero_cat


class RetrievalAUROC(RetrievalMetric):
    """AUROC of each query's top ``top_k`` documents, aggregated over the queries (reference retrieval/auroc.py);
    ``max_fpr`` gives the McClish-standardised partial area up to that false positive rate."""

    is_differentiable: bool = False
    higher_is_better: bool = True
    full_state_update: bool = False
    plot_lower_bound: float = 0.0
    plot_upper_bound: float = 1.0

    def __init__(
        self,
        empty_target_action: Literal["error", "skip", "neg", "pos"] = "neg",
        ignore_index: Optional[int] = None,
        top_k: Optional[int] = None,
        max_fpr: Optional[float] = None,
        aggregation: Union[Literal["mean", "median", "min", "max"], Callable] = "mean",
        **kwargs: Any,
    ) -> None:
        super().__init__(empty_target_action=empty_target_action, ignore_index=ignore_index, aggregation=aggregation, **kwargs)
        if top_k is not None and not (isinstance(top_k, int) and top_k > 0):
            raise ValueError("`top_k` has to be a positive integer or None")
        self.top_k = top_k
        if max_fpr is not None and not isinstance(max_fpr, float) and 0 < max_fpr <= 1:
            raise ValueError(f"Arguments `max_fpr` should be a float in range (0, 1], but got: {max_fpr}")
        self.max_fpr = max_fpr

    def _evaluate(self, groups: "_native.RetrievalGroups") -> "tuple[Tensor, Tensor]":
        _check_max_fpr(self.max_fpr)
        return _native.retrieval_auroc(groups, self.top_k, self.max_fpr)

    def _metric(self, preds: Tensor, target: Tensor) -> Tensor:
        return retrieval_auroc(preds, target, top_k=self.top_k, max_fpr=self.max_fpr)


class RetrievalPrecisionRecallCurve(RetrievalMetric):
    """Precision and recall at k = 1..``max_k``, aggregated over the queries, and the k (reference
    retrieval/precision_recall_curve.py).  ``max_k=None`` takes the longest query.  Unlike the reference's class, which
    is a plain ``Metric``, this one is a ``RetrievalMetric``: it shares the group sort of a compute group."""

    is_differentiable: bool = False
    higher_is_better: bool = True
    full_state_update: bool = False

    def __init__(
        self,
        max_k: Optional[int] = None,
        adaptive_k: bool = False,
        empty_target_action: str = "neg",
        ignore_index: Optional[int] = None,
        aggregation: Union[Literal["mean", "median", "min", "max"], Callable] = "mean",
        **kwargs: Any,
    ) -> None:
        super().__init__(empty_target_action=empty_target_action, ignore_index=ignore_index, aggregation=aggregation, **kwargs)
        if (max_k is not None) and not (isinstance(max_k, int) and max_k > 0):
            raise ValueError("`max_k` has to be a positive integer or None")
        self.max_k = max_k
        if not isinstance(adaptive_k, bool):
            raise ValueError("`adaptive_k` has to be a boolean")
        self.adaptive_k = adaptive_k

    def compute(self) -> "tuple[Tensor, Tensor, Tensor]":
        """``(precision [max_k], recall [max_k], top_k [max_k])``: one K16f launch for every query's row, then the empty
        rows' action and the aggregation over the rows."""
        preds = dim_zero_cat(self.preds)
        groups = self._groups()
        max_k = self.max_k
        if max_k is None:  # the longest query: one host read
            q = groups.num_queries
            max_k = int((groups.offsets[1:q + 1] - groups.offsets[:q]).max())
        precision, recall, empty = _native.retrieval_pr_curve(groups, max_k, self.adaptive_k)
        action = self.empty_target_action
        if action == "error":
            if bool(empty.any()):
                raise ValueError(self._empty_message)
        elif action == "skip":
            precision, recall = precision[~empty], recall[~empty]
        elif action == "pos":
            precision = torch.where(empty[:, None], torch.ones_like(precision), precision)
            recall = torch.where(empty[:, None], torch.ones_like(recall), recall)
        if precision.shape[0]:
            precision = _retrieval_aggregate(precision.to(preds), aggregation=self.aggregation, dim=0)
            recall = _retrieval_aggregate(recall.to(preds), aggregation=self.aggregation, dim=0)
        else:
            precision, recall = torch.zeros(max_k).to(preds), torch.zeros(max_k).to(preds)
        return precision, recall, torch.arange(1, max_k + 1, device=preds.device)

    def _metric(self, preds: Tensor, target: Tensor) -> Tensor:
        return retrieval_precision_recall_curve(preds, target, self.max_k, self.adaptive_k)


class RetrievalRecallAtFixedPrecision(RetrievalPrecisionRecallCurve):
    """The largest recall whose precision is at least ``min_precision`` on the aggregated curve, and its k (reference
    retrieval/precision_recall_curve.py); ``(0, max_k)`` when no k qualifies or the largest recall is 0."""

    higher_is_better = True

    def __init__(
        self,
        min_precision: float = 0.0,
        max_k: Optional[int] = None,
        adaptive_k: bool = False,
        empty_target_action: str = "neg",
        ignore_index: Optional[int] = None,
        **kwargs: Any,
    ) -> None:
        super().__init__(max_k=max_k, adaptive_k=adaptive_k, empty_target_action=empty_target_action,
                         ignore_index=ignore_index, **kwargs)
        if not (isinstance(min_precision, float) and 0.0 <= min_precision <= 1.0):
            raise ValueError("`min_precision` has to be a positive float between 0 and 1")
        self.min_precision = min_precision

    def compute(self) -> "tuple[Tensor, Tensor]":  # type: ignore[override]
        """Device ops only: no host read beyond the curve's.  Ties in recall go to the largest k, as the reference's
        ``max`` over ``(recall, k)`` pairs does."""
        precision, recall, top_k = super().compute()
        cand = torch.where(precision >= self.min_precision, recall, torch.full_like(recall, -1.0))
        best = cand.max()
        best_k = torch.where(cand == best, top_k, torch.zeros_like(top_k)).max()
        none = best <= 0.0  # nothing qualifies (-1), or the largest recall is 0
        max_recall = torch.where(none, torch.zeros_like(best), best)
        best_k = torch.where(none, torch.full_like(best_k, top_k.numel()), best_k)
        return max_recall, best_k
