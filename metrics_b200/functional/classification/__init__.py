"""Functional classification metrics (reference: src/torchmetrics/functional/classification/)."""
from metrics_b200.functional.classification.accuracy import multiclass_accuracy  # noqa: F401
from metrics_b200.functional.classification.confusion_matrix import multiclass_confusion_matrix  # noqa: F401
from metrics_b200.functional.classification.f_beta import multiclass_f1_score, multiclass_fbeta_score  # noqa: F401
from metrics_b200.functional.classification.stat_scores import multiclass_stat_scores  # noqa: F401
from metrics_b200.functional.classification.auroc import binary_auroc, multiclass_auroc  # noqa: F401,E402
from metrics_b200.functional.classification.average_precision import (  # noqa: F401,E402
    binary_average_precision,
    multiclass_average_precision,
)
from metrics_b200.functional.classification.precision_recall_curve import (  # noqa: F401,E402
    binary_precision_recall_curve,
    multiclass_precision_recall_curve,
)
from metrics_b200.functional.classification.roc import binary_roc, multiclass_roc  # noqa: F401,E402
from metrics_b200.functional.classification.accuracy import binary_accuracy, multilabel_accuracy  # noqa: F401,E402
from metrics_b200.functional.classification.confusion_matrix import (  # noqa: F401,E402
    binary_confusion_matrix,
    confusion_matrix,
    multilabel_confusion_matrix,
)
from metrics_b200.functional.classification.f_beta import (  # noqa: F401,E402
    binary_f1_score,
    binary_fbeta_score,
    multilabel_f1_score,
    multilabel_fbeta_score,
)
from metrics_b200.functional.classification.stat_scores import (  # noqa: F401,E402
    binary_stat_scores,
    multilabel_stat_scores,
    stat_scores,
)
from metrics_b200.functional.classification.auroc import multilabel_auroc  # noqa: F401,E402
from metrics_b200.functional.classification.average_precision import multilabel_average_precision  # noqa: F401,E402
from metrics_b200.functional.classification.precision_recall_curve import multilabel_precision_recall_curve  # noqa: F401,E402
from metrics_b200.functional.classification.roc import multilabel_roc  # noqa: F401,E402
from metrics_b200.functional.classification.ratio_metrics import (  # noqa: F401,E402
    binary_hamming_distance,
    binary_negative_predictive_value,
    binary_precision,
    binary_recall,
    binary_specificity,
    hamming_distance,
    multiclass_hamming_distance,
    multiclass_negative_predictive_value,
    multiclass_precision,
    multiclass_recall,
    multiclass_specificity,
    multilabel_hamming_distance,
    multilabel_negative_predictive_value,
    multilabel_precision,
    multilabel_recall,
    multilabel_specificity,
    negative_predictive_value,
    precision,
    recall,
    specificity,
)
from metrics_b200.functional.classification.confmat_metrics import (  # noqa: F401,E402
    binary_cohen_kappa,
    binary_jaccard_index,
    binary_matthews_corrcoef,
    multiclass_cohen_kappa,
    multiclass_jaccard_index,
    multiclass_matthews_corrcoef,
    multilabel_jaccard_index,
    multilabel_matthews_corrcoef,
)
from metrics_b200.functional.classification.at_fixed import (  # noqa: F401,E402
    binary_precision_at_fixed_recall,
    binary_recall_at_fixed_precision,
    binary_sensitivity_at_specificity,
    binary_specificity_at_sensitivity,
    multiclass_precision_at_fixed_recall,
    multiclass_recall_at_fixed_precision,
    multiclass_sensitivity_at_specificity,
    multiclass_specificity_at_sensitivity,
    multilabel_precision_at_fixed_recall,
    multilabel_recall_at_fixed_precision,
    multilabel_sensitivity_at_specificity,
    multilabel_specificity_at_sensitivity,
)
from metrics_b200.functional.classification.exact_match import exact_match, multiclass_exact_match, multilabel_exact_match  # noqa: F401,E402
from metrics_b200.functional.classification.logauc import binary_logauc, logauc, multiclass_logauc, multilabel_logauc  # noqa: F401,E402
from metrics_b200.functional.classification.group_fairness import (  # noqa: F401,E402
    binary_fairness,
    binary_groups_stat_rates,
    demographic_parity,
    equal_opportunity,
)
from metrics_b200.functional.classification.accuracy import accuracy  # noqa: F401,E402
from metrics_b200.functional.classification.auroc import auroc  # noqa: F401,E402
from metrics_b200.functional.classification.average_precision import average_precision  # noqa: F401,E402
from metrics_b200.functional.classification.roc import roc  # noqa: F401,E402
from metrics_b200.functional.classification.precision_recall_curve import precision_recall_curve  # noqa: F401,E402
from metrics_b200.functional.classification.f_beta import f1_score, fbeta_score  # noqa: F401,E402
from metrics_b200.functional.classification.confmat_metrics import cohen_kappa, jaccard_index, matthews_corrcoef  # noqa: F401,E402
from metrics_b200.functional.classification.at_fixed import (  # noqa: F401,E402
    precision_at_fixed_recall,
    recall_at_fixed_precision,
    sensitivity_at_specificity,
    specificity_at_sensitivity,
)
from metrics_b200.functional.classification.calibration_error import (  # noqa: F401,E402
    binary_calibration_error,
    calibration_error,
    multiclass_calibration_error,
)

# The reference's import paths `<package>.{cohen_kappa, matthews_corrcoef, negative_predictive_value, specificity}` are alias submodules that share a name with a function exported
# above.  Loading a submodule binds it as a package attribute, so load them now and re-bind the functions afterwards: a
# later `import` of an already-loaded submodule does not touch the attribute again.
import importlib as _importlib  # noqa: E402

for _name in ("cohen_kappa", "matthews_corrcoef", "negative_predictive_value", "specificity"):
    _fn = globals()[_name]
    _importlib.import_module(f"{__name__}.{_name}")
    globals()[_name] = _fn
del _importlib, _name, _fn
