"""Modular classification metrics (reference: src/torchmetrics/classification/)."""
from metrics_b200.classification.accuracy import MulticlassAccuracy  # noqa: F401
from metrics_b200.classification.confusion_matrix import MulticlassConfusionMatrix  # noqa: F401
from metrics_b200.classification.f_beta import MulticlassF1Score, MulticlassFBetaScore  # noqa: F401
from metrics_b200.classification.stat_scores import MulticlassStatScores  # noqa: F401
from metrics_b200.classification.auroc import BinaryAUROC, MulticlassAUROC  # noqa: F401,E402
from metrics_b200.classification.average_precision import BinaryAveragePrecision, MulticlassAveragePrecision  # noqa: F401,E402
from metrics_b200.classification.precision_recall_curve import (  # noqa: F401,E402
    BinaryPrecisionRecallCurve,
    MulticlassPrecisionRecallCurve,
)
from metrics_b200.classification.roc import BinaryROC, MulticlassROC  # noqa: F401,E402
from metrics_b200.classification.accuracy import Accuracy, BinaryAccuracy, MultilabelAccuracy  # noqa: F401,E402
from metrics_b200.classification.confusion_matrix import (  # noqa: F401,E402
    BinaryConfusionMatrix,
    ConfusionMatrix,
    MultilabelConfusionMatrix,
)
from metrics_b200.classification.f_beta import (  # noqa: F401,E402
    BinaryF1Score,
    BinaryFBetaScore,
    F1Score,
    FBetaScore,
    MultilabelF1Score,
    MultilabelFBetaScore,
)
from metrics_b200.classification.stat_scores import BinaryStatScores, MultilabelStatScores, StatScores  # noqa: F401,E402
from metrics_b200.classification.auroc import AUROC  # noqa: F401,E402
from metrics_b200.classification.average_precision import AveragePrecision  # noqa: F401,E402
from metrics_b200.classification.precision_recall_curve import PrecisionRecallCurve  # noqa: F401,E402
from metrics_b200.classification.roc import ROC  # noqa: F401,E402
from metrics_b200.classification.auroc import MultilabelAUROC  # noqa: F401,E402
from metrics_b200.classification.average_precision import MultilabelAveragePrecision  # noqa: F401,E402
from metrics_b200.classification.precision_recall_curve import MultilabelPrecisionRecallCurve  # noqa: F401,E402
from metrics_b200.classification.roc import MultilabelROC  # noqa: F401,E402
from metrics_b200.classification.ratio_metrics import (  # noqa: F401,E402
    BinaryHammingDistance,
    BinaryNegativePredictiveValue,
    BinaryPrecision,
    BinaryRecall,
    BinarySpecificity,
    HammingDistance,
    MulticlassHammingDistance,
    MulticlassNegativePredictiveValue,
    MulticlassPrecision,
    MulticlassRecall,
    MulticlassSpecificity,
    MultilabelHammingDistance,
    MultilabelNegativePredictiveValue,
    MultilabelPrecision,
    MultilabelRecall,
    MultilabelSpecificity,
    NegativePredictiveValue,
    Precision,
    Recall,
    Specificity,
)
from metrics_b200.classification.confmat_metrics import (  # noqa: F401,E402
    BinaryCohenKappa,
    BinaryJaccardIndex,
    BinaryMatthewsCorrCoef,
    CohenKappa,
    JaccardIndex,
    MatthewsCorrCoef,
    MulticlassCohenKappa,
    MulticlassJaccardIndex,
    MulticlassMatthewsCorrCoef,
    MultilabelJaccardIndex,
    MultilabelMatthewsCorrCoef,
)
from metrics_b200.classification.at_fixed import (  # noqa: F401,E402
    BinaryPrecisionAtFixedRecall,
    BinaryRecallAtFixedPrecision,
    BinarySensitivityAtSpecificity,
    BinarySpecificityAtSensitivity,
    MulticlassPrecisionAtFixedRecall,
    MulticlassRecallAtFixedPrecision,
    MulticlassSensitivityAtSpecificity,
    MulticlassSpecificityAtSensitivity,
    MultilabelPrecisionAtFixedRecall,
    MultilabelRecallAtFixedPrecision,
    MultilabelSensitivityAtSpecificity,
    MultilabelSpecificityAtSensitivity,
    PrecisionAtFixedRecall,
    RecallAtFixedPrecision,
    SensitivityAtSpecificity,
    SpecificityAtSensitivity,
)
from metrics_b200.classification.exact_match import ExactMatch, MulticlassExactMatch, MultilabelExactMatch  # noqa: F401,E402
from metrics_b200.classification.logauc import BinaryLogAUC, LogAUC, MulticlassLogAUC, MultilabelLogAUC  # noqa: F401,E402
from metrics_b200.classification.group_fairness import BinaryFairness, BinaryGroupStatRates  # noqa: F401,E402
from metrics_b200.classification.calibration_error import (  # noqa: F401,E402
    BinaryCalibrationError,
    CalibrationError,
    MulticlassCalibrationError,
)
