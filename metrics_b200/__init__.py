"""metrics_b200 — the TorchMetrics update()/compute()/sync hot path, rebuilt for H100 (sm_90a).

Drop-in for the reference's `Metric` / `MetricCollection` API and the classification / detection / regression
metric families named in DESIGN.md; every per-batch `_update` runs in a hand-written CUDA kernel reached through
the C-ABI in `include/metrics_b200.h` (there is no CPU fallback: inputs must be CUDA tensors).
"""
from metrics_b200.metric import CompositionalMetric, Metric  # noqa: F401  (first: the metric packages below need it)
from metrics_b200.collections import MetricCollection  # noqa: F401
from metrics_b200 import functional  # noqa: F401
from metrics_b200.classification import (  # noqa: F401  (reference __init__.py:56-83, the rows on the path)
    AUROC,
    ROC,
    Accuracy,
    AveragePrecision,
    CohenKappa,
    ConfusionMatrix,
    ExactMatch,
    F1Score,
    FBetaScore,
    HammingDistance,
    JaccardIndex,
    LogAUC,
    MatthewsCorrCoef,
    NegativePredictiveValue,
    Precision,
    PrecisionAtFixedRecall,
    PrecisionRecallCurve,
    Recall,
    RecallAtFixedPrecision,
    SensitivityAtSpecificity,
    Specificity,
    SpecificityAtSensitivity,
    StatScores,
)
from metrics_b200.regression import (  # noqa: F401  (reference __init__.py:113-134)
    CriticalSuccessIndex,
    ExplainedVariance,
    KendallRankCorrCoef,
    KLDivergence,
    LogCoshError,
    MeanAbsoluteError,
    MeanAbsolutePercentageError,
    MeanSquaredError,
    MeanSquaredLogError,
    MinkowskiDistance,
    R2Score,
    RelativeSquaredError,
    SpearmanCorrCoef,
    SymmetricMeanAbsolutePercentageError,
    TweedieDevianceScore,
    WeightedMeanAbsolutePercentageError,
)
from metrics_b200.wrappers import ClasswiseWrapper  # noqa: F401

__version__ = "0.1.0"
__all__ = [_n for _n in dir() if not _n.startswith("_")]
