"""Functional retrieval metrics (reference: src/torchmetrics/functional/retrieval/), on kernel K16: the eight per-query
metrics on K16d, `retrieval_auroc` on K16e and `retrieval_precision_recall_curve` on K16f."""
from metrics_b200.functional.retrieval._curves import retrieval_auroc, retrieval_precision_recall_curve
from metrics_b200.functional.retrieval._metrics import (
    retrieval_average_precision,
    retrieval_fall_out,
    retrieval_hit_rate,
    retrieval_normalized_dcg,
    retrieval_precision,
    retrieval_r_precision,
    retrieval_recall,
    retrieval_reciprocal_rank,
)

__all__ = [
    "retrieval_auroc",
    "retrieval_average_precision",
    "retrieval_fall_out",
    "retrieval_hit_rate",
    "retrieval_normalized_dcg",
    "retrieval_precision",
    "retrieval_precision_recall_curve",
    "retrieval_r_precision",
    "retrieval_recall",
    "retrieval_reciprocal_rank",
]
