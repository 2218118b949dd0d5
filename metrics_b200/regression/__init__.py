"""Modular regression metrics (reference: src/torchmetrics/regression/)."""
from metrics_b200.regression.metrics import (  # noqa: F401
    CriticalSuccessIndex,
    ExplainedVariance,
    LogCoshError,
    MeanAbsoluteError,
    MeanAbsolutePercentageError,
    MeanSquaredError,
    MeanSquaredLogError,
    MinkowskiDistance,
    R2Score,
    RelativeSquaredError,
    SymmetricMeanAbsolutePercentageError,
    TweedieDevianceScore,
    WeightedMeanAbsolutePercentageError,
)
from metrics_b200.regression.kl_divergence import KLDivergence  # noqa: F401,E402
from metrics_b200.regression.kendall import KendallRankCorrCoef  # noqa: F401,E402
from metrics_b200.regression.spearman import SpearmanCorrCoef  # noqa: F401,E402
