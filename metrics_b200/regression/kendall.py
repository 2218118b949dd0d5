"""KendallRankCorrCoef (reference: regression/kendall.py:36-170).  List states `preds` / `target` ("cat", not persistent,
``[N, 1]`` per batch for one output) as in the reference; `compute()` counts the pairs in the rank-correlation kernel K17."""

from typing import Any, List, Optional, Union

from torch import Tensor
from typing_extensions import Literal

from metrics_b200.functional.regression.kendall import (
    _kendall_corrcoef_compute,
    _kendall_corrcoef_update,
    _MetricVariant,
    _TestAlternative,
)
from metrics_b200.metric import Metric
from metrics_b200.utilities.data import dim_zero_cat


class KendallRankCorrCoef(Metric):
    """Kendall's rank correlation coefficient tau (variant "a", "b" or "c") over every batch seen, per output column, and the
    p-value of its t-test when ``t_test``."""

    is_differentiable = False
    higher_is_better = None
    full_state_update = True
    plot_lower_bound: float = 0.0
    plot_upper_bound: float = 1.0

    preds: List[Tensor]
    target: List[Tensor]

    def __init__(
        self,
        variant: Literal["a", "b", "c"] = "b",
        t_test: bool = False,
        alternative: Optional[Literal["two-sided", "less", "greater"]] = "two-sided",
        num_outputs: int = 1,
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        if not isinstance(t_test, bool):
            raise ValueError(f"Argument `t_test` is expected to be of a type `bool`, but got {type(t_test)}.")
        if t_test and alternative is None:
            raise ValueError("Argument `alternative` is required if `t_test=True` but got `None`.")

        self.variant = _MetricVariant.from_str(str(variant))
        self.alternative = _TestAlternative.from_str(str(alternative)) if t_test else None
        self.num_outputs = num_outputs

        self.add_state("preds", [], dist_reduce_fx="cat")
        self.add_state("target", [], dist_reduce_fx="cat")

    def update(self, preds: Tensor, target: Tensor) -> None:
        self.preds, self.target = _kendall_corrcoef_update(preds, target, self.preds, self.target, num_outputs=self.num_outputs)

    def compute(self) -> Union[Tensor, tuple[Tensor, Tensor]]:
        tau, p_value = _kendall_corrcoef_compute(dim_zero_cat(self.preds), dim_zero_cat(self.target), self.variant,
                                                 self.alternative)
        if p_value is not None:
            return tau, p_value
        return tau
