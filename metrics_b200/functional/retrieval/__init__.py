"""Functional retrieval metrics (reference: src/torchmetrics/functional/retrieval/), on kernel K16.
`retrieval_auroc` and `retrieval_precision_recall_curve` are not implemented yet (DESIGN.md section 0)."""
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
    "retrieval_average_precision",
    "retrieval_fall_out",
    "retrieval_hit_rate",
    "retrieval_normalized_dcg",
    "retrieval_precision",
    "retrieval_r_precision",
    "retrieval_recall",
    "retrieval_reciprocal_rank",
]
