"""Dice score, modular (reference: segmentation/dice.py)."""
from typing import Any, List, Optional

from torch import Tensor
from typing_extensions import Literal

from metrics_b200.functional.segmentation.dice import _dice_score_compute, _dice_score_update, _dice_score_validate_args
from metrics_b200.metric import Metric
from metrics_b200.utilities.data import dim_zero_cat


class DiceScore(Metric):
    r"""Dice score for semantic segmentation (reference :34-143).

    ``preds`` / ``target``: one-hot ``(N, C, ...)`` tensors (bool, integer, float32 / float16 / bfloat16), or int64 class
    indices ``(N, ...)`` with ``input_format="index"``.  Each update appends the per-sample, per-class ``2 * intersection``,
    ``pred_sum + target_sum`` and ``target_sum`` to the ``cat`` states; ``compute`` averages the dice score over the
    samples.  The counts of an update come from one read of the inputs (kernel K15)."""

    full_state_update: bool = False
    is_differentiable: bool = False
    higher_is_better: bool = True
    plot_lower_bound: float = 0.0
    plot_upper_bound: float = 1.0

    numerator: List[Tensor]
    denominator: List[Tensor]
    support: List[Tensor]

    def __init__(
        self,
        num_classes: int,
        include_background: bool = True,
        average: Optional[Literal["micro", "macro", "weighted", "none"]] = "micro",
        input_format: Literal["one-hot", "index"] = "one-hot",
        **kwargs: Any,
    ) -> None:
        super().__init__(**kwargs)
        _dice_score_validate_args(num_classes, include_background, average, input_format)
        self.num_classes = num_classes
        self.include_background = include_background
        self.average = average
        self.input_format = input_format

        self.add_state("numerator", [], dist_reduce_fx="cat")
        self.add_state("denominator", [], dist_reduce_fx="cat")
        self.add_state("support", [], dist_reduce_fx="cat")

    def update(self, preds: Tensor, target: Tensor) -> None:
        """Update the state with new data."""
        numerator, denominator, support = _dice_score_update(
            preds, target, self.num_classes, self.include_background, self.input_format
        )
        self.numerator.append(numerator)
        self.denominator.append(denominator)
        self.support.append(support)

    def compute(self) -> Tensor:
        """Computes the Dice Score."""
        return _dice_score_compute(
            dim_zero_cat(self.numerator),
            dim_zero_cat(self.denominator),
            self.average,
            support=dim_zero_cat(self.support) if self.average == "weighted" else None,
        ).mean(dim=0)
