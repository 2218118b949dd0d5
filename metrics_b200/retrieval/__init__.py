"""Retrieval metrics (reference: src/torchmetrics/retrieval/), on kernel K16.  `RetrievalAUROC`,
`RetrievalPrecisionRecallCurve` and `RetrievalRecallAtFixedPrecision` are not implemented yet (DESIGN.md section 0)."""
from metrics_b200.retrieval.base import RetrievalMetric, _retrieval_aggregate
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
    "RetrievalFallOut",
    "RetrievalHitRate",
    "RetrievalMAP",
    "RetrievalMRR",
    "RetrievalNormalizedDCG",
    "RetrievalPrecision",
    "RetrievalRPrecision",
    "RetrievalRecall",
]
