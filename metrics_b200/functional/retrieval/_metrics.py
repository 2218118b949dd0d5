"""Retrieval metrics of one query (reference: src/torchmetrics/functional/retrieval/).  The whole input is one query: one
group sort and one evaluation launch of kernel K16 (``_native.retrieval_*``); the argument checks run first, as in the
reference, so they raise the reference's errors at the same call."""
from typing import Optional

from torch import Tensor

from metrics_b200 import _native
from metrics_b200.utilities.checks import _check_retrieval_functional_inputs


_FLOAT_R_MESSAGE = "only integer tensors of a single element can be converted to an index"


def _one_query(preds: Tensor, target: Tensor, kind: int, top_k: Optional[int] = None, adaptive_k: bool = False) -> Tensor:
    groups = _native.retrieval_sort(None, preds, target)
    ideal = _native.retrieval_sort_ideal(groups) if kind == _native.RET_NDCG else None
    value, _ = _native.retrieval_evaluate(groups, kind, top_k, adaptive_k, ideal)
    return value[0]


def _positive_top_k(top_k: Optional[int], n: int) -> int:
    top_k = n if top_k is None else top_k
    if not (isinstance(top_k, int) and top_k > 0):
        raise ValueError("`top_k` has to be a positive integer or None")
    return top_k


def retrieval_average_precision(preds: Tensor, target: Tensor, top_k: Optional[int] = None) -> Tensor:
    """Average precision of one query over its top ``top_k`` documents (reference average_precision.py)."""
    preds, target = _check_retrieval_functional_inputs(preds, target)
    top_k = top_k or preds.shape[-1]
    if not isinstance(top_k, int) and top_k <= 0:
        raise ValueError(f"Argument ``top_k`` has to be a positive integer or None, but got {top_k}.")
    return _one_query(preds, target, _native.RET_AP, top_k)


def retrieval_reciprocal_rank(preds: Tensor, target: Tensor, top_k: Optional[int] = None) -> Tensor:
    """Reciprocal rank of the first relevant document within the top ``top_k`` (reference reciprocal_rank.py)."""
    preds, target = _check_retrieval_functional_inputs(preds, target)
    top_k = top_k or preds.shape[-1]
    if not isinstance(top_k, int) and top_k <= 0:
        raise ValueError(f"Argument ``top_k`` has to be a positive integer or None, but got {top_k}.")
    return _one_query(preds, target, _native.RET_RR, top_k)


def retrieval_precision(preds: Tensor, target: Tensor, top_k: Optional[int] = None, adaptive_k: bool = False) -> Tensor:
    """Fraction of relevant documents among the top ``top_k`` (reference precision.py)."""
    preds, target = _check_retrieval_functional_inputs(preds, target)
    if not isinstance(adaptive_k, bool):
        raise ValueError("`adaptive_k` has to be a boolean")
    if top_k is None or (adaptive_k and top_k > preds.shape[-1]):
        top_k = preds.shape[-1]
    if not (isinstance(top_k, int) and top_k > 0):
        raise ValueError("`top_k` has to be a positive integer or None")
    return _one_query(preds, target, _native.RET_PRECISION, top_k, adaptive_k)


def retrieval_recall(preds: Tensor, target: Tensor, top_k: Optional[int] = None) -> Tensor:
    """Fraction of the relevant documents found in the top ``top_k`` (reference recall.py)."""
    preds, target = _check_retrieval_functional_inputs(preds, target)
    return _one_query(preds, target, _native.RET_RECALL, _positive_top_k(top_k, preds.shape[-1]))


def retrieval_hit_rate(preds: Tensor, target: Tensor, top_k: Optional[int] = None) -> Tensor:
    """1 when a relevant document is in the top ``top_k``, else 0 (reference hit_rate.py)."""
    preds, target = _check_retrieval_functional_inputs(preds, target)
    return _one_query(preds, target, _native.RET_HIT_RATE, _positive_top_k(top_k, preds.shape[-1]))


def retrieval_fall_out(preds: Tensor, target: Tensor, top_k: Optional[int] = None) -> Tensor:
    """Fraction of the non-relevant documents found in the top ``top_k`` (reference fall_out.py)."""
    preds, target = _check_retrieval_functional_inputs(preds, target)
    return _one_query(preds, target, _native.RET_FALL_OUT, _positive_top_k(top_k, preds.shape[-1]))


def retrieval_r_precision(preds: Tensor, target: Tensor) -> Tensor:
    """Precision over the top R documents, R = number of relevant ones (reference r_precision.py)."""
    preds, target = _check_retrieval_functional_inputs(preds, target)
    if target.is_floating_point() and bool(target.sum()):  # the reference slices the ranking with the float sum
        raise TypeError(_FLOAT_R_MESSAGE)
    return _one_query(preds, target, _native.RET_R_PRECISION)


def retrieval_normalized_dcg(preds: Tensor, target: Tensor, top_k: Optional[int] = None) -> Tensor:
    """Normalized discounted cumulative gain with graded targets, score ties averaged (reference ndcg.py)."""
    preds, target = _check_retrieval_functional_inputs(preds, target, allow_non_binary_target=True)
    return _one_query(preds, target, _native.RET_NDCG, _positive_top_k(top_k, preds.shape[-1]))
