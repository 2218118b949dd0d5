"""SpearmanCorrCoef (reference: regression/spearman.py:30-108).  List states `preds` / `target` ("cat", not persistent) as in
the reference; `compute()` ranks the concatenated columns in the rank-correlation kernel K17."""
from typing import Any, List
from torch import Tensor
from metrics_b200.functional.regression.spearman import _spearman_corrcoef_compute, _spearman_corrcoef_update
from metrics_b200.metric import Metric
from metrics_b200.utilities.data import dim_zero_cat
from metrics_b200.utilities.prints import rank_zero_warn
class SpearmanCorrCoef(Metric):
    """Spearman's rank correlation coefficient over every batch seen, per output column."""
    is_differentiable: bool = False
    higher_is_better: bool = True
    full_state_update: bool = False
    plot_lower_bound: float = -1.0
    plot_upper_bound: float = 1.0
    preds: List[Tensor]
    target: List[Tensor]
    def __init__(self, num_outputs: int = 1, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        rank_zero_warn(
            "Metric `SpearmanCorrcoef` will save all targets and predictions in the buffer."
            " For large datasets, this may lead to large memory footprint."
        )
        if not isinstance(num_outputs, int) and num_outputs < 1:
            raise ValueError(f"Expected argument `num_outputs` to be an int larger than 0, but got {num_outputs}")
        self.num_outputs = num_outputs
        self.add_state("preds", default=[], dist_reduce_fx="cat")
        self.add_state("target", default=[], dist_reduce_fx="cat")
    def update(self, preds: Tensor, target: Tensor) -> None:
        preds, target = _spearman_corrcoef_update(preds, target, num_outputs=self.num_outputs)
        self.preds.append(preds.to(self.dtype))
        self.target.append(target.to(self.dtype))
    def compute(self) -> Tensor:
        return _spearman_corrcoef_compute(dim_zero_cat(self.preds), dim_zero_cat(self.target))
