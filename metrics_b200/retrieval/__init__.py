"""Retrieval metrics (reference: src/torchmetrics/retrieval/), on kernel K16: one group sort per compute group, then one
evaluation launch per metric.  The deprecated aliases of the reference are not provided (DESIGN.md section 0)."""
from metrics_b200.retrieval.base import RetrievalMetric, _retrieval_aggregate
from metrics_b200.retrieval.curves import RetrievalAUROC, RetrievalPrecisionRecallCurve, RetrievalRecallAtFixedPrecision
from metrics_b200.retrieval.metrics import (
    RetrievalFallOut,
    RetrievalHitRate,
    RetrievalMAP,
    RetrievalMRR,
    RetrievalNormalizedDCG,
    RetrievalPrecision,
    RetrievalRecall,
    RetrievalRPrecision,
)

__all__ = [
    "RetrievalAUROC",
    "RetrievalFallOut",
    "RetrievalHitRate",
    "RetrievalMAP",
    "RetrievalMRR",
    "RetrievalNormalizedDCG",
    "RetrievalPrecision",
    "RetrievalPrecisionRecallCurve",
    "RetrievalRPrecision",
    "RetrievalRecall",
    "RetrievalRecallAtFixedPrecision",
]
