"""Functional regression metrics (reference: src/torchmetrics/functional/regression/)."""
from metrics_b200.functional.regression.metrics import (  # noqa: F401
    critical_success_index,
    explained_variance,
    log_cosh_error,
    mean_absolute_error,
    mean_absolute_percentage_error,
    mean_squared_error,
    mean_squared_log_error,
    minkowski_distance,
    r2_score,
    relative_squared_error,
    symmetric_mean_absolute_percentage_error,
    tweedie_deviance_score,
    weighted_mean_absolute_percentage_error,
)

from metrics_b200.functional.regression.kl_divergence import kl_divergence  # noqa: F401,E402
from metrics_b200.functional.regression.kendall import kendall_rank_corrcoef  # noqa: F401,E402
from metrics_b200.functional.regression.spearman import spearman_corrcoef  # noqa: F401,E402

# The reference's import paths `<package>.{explained_variance}` are alias submodules that share a name with a function exported
# above.  Loading a submodule binds it as a package attribute, so load them now and re-bind the functions afterwards: a
# later `import` of an already-loaded submodule does not touch the attribute again.
import importlib as _importlib  # noqa: E402

for _name in ("explained_variance", "kl_divergence"):
    _fn = globals()[_name]
    _importlib.import_module(f"{__name__}.{_name}")
    globals()[_name] = _fn
del _importlib, _name, _fn
