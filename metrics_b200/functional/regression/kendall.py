"""Kendall's rank correlation (reference: functional/regression/kendall.py).  The reference compares every row with all later
rows in a Python loop; here the rank-correlation kernel K17 (`mb200_kendall_rank_corrcoef`, csrc/rankcorr.cu) counts the
concordant and discordant pairs exactly in O(n log n) and computes tau and the t-test on the device."""
from __future__ import annotations

from typing import List, Optional, Union

from torch import Tensor
from typing_extensions import Literal

from metrics_b200 import _native
from metrics_b200.functional.regression.utils import _check_data_shape_to_num_outputs
from metrics_b200.utilities.checks import _check_same_shape
from metrics_b200.utilities.data import dim_zero_cat
from metrics_b200.utilities.enums import EnumStr


class _MetricVariant(EnumStr):
    """Variants of Kendall's tau."""

    A = "a"
    B = "b"
    C = "c"

    @staticmethod
    def _name() -> str:
        return "variant"


class _TestAlternative(EnumStr):
    """Alternative hypotheses of the t-test."""

    TWO_SIDED = "two-sided"
    LESS = "less"
    GREATER = "greater"

    @staticmethod
    def _name() -> str:
        return "alternative"


def _kendall_corrcoef_update(
    preds: Tensor,
    target: Tensor,
    concat_preds: Optional[List[Tensor]] = None,
    concat_target: Optional[List[Tensor]] = None,
    num_outputs: int = 1,
) -> tuple[List[Tensor], List[Tensor]]:
    """Check the inputs and append them to the lists (reference :225-258); one output is stored as ``[N, 1]``."""
    concat_preds = concat_preds or []
    concat_target = concat_target or []
    _check_same_shape(preds, target)
    _check_data_shape_to_num_outputs(preds, target, num_outputs)
    if num_outputs == 1:
        preds = preds.unsqueeze(1)
        target = target.unsqueeze(1)
    concat_preds.append(preds)
    concat_target.append(target)
    return concat_preds, concat_target


def _kendall_corrcoef_compute(
    preds: Tensor,
    target: Tensor,
    variant: _MetricVariant,
    alternative: Optional[_TestAlternative] = None,
) -> tuple[Tensor, Optional[Tensor]]:
    """Tau of ``variant`` per column and, with an ``alternative``, the p-value of its asymptotic t-test (reference :261-318).
    float32; scalars for one column.  Pair counts and tie terms are exact (deviation from the reference, whose int64 tau-b
    denominator overflows past about 78 000 rows)."""
    if not isinstance(variant, _MetricVariant):
        variant = _MetricVariant.from_str(str(variant))
    if alternative is not None and not isinstance(alternative, _TestAlternative):
        alternative = _TestAlternative.from_str(str(alternative))
    return _native.kendall_rank_corrcoef(preds, target, variant.value, None if alternative is None else alternative.value)


def kendall_rank_corrcoef(
    preds: Tensor,
    target: Tensor,
    variant: Literal["a", "b", "c"] = "b",
    t_test: bool = False,
    alternative: Optional[Literal["two-sided", "less", "greater"]] = "two-sided",
) -> Union[Tensor, tuple[Tensor, Tensor]]:
    """Kendall's rank correlation coefficient tau of ``preds`` and ``target`` (``[N]`` or ``[N, d]``), and the p-value of its
    t-test when ``t_test`` (reference :321-416)."""
    if not isinstance(t_test, bool):
        raise ValueError(f"Argument `t_test` is expected to be of a type `bool`, but got {type(t_test)}.")
    if t_test and alternative is None:
        raise ValueError("Argument `alternative` is required if `t_test=True` but got `None`.")

    _variant = _MetricVariant.from_str(str(variant))
    _alternative = _TestAlternative.from_str(str(alternative)) if t_test else None

    _preds, _target = _kendall_corrcoef_update(
        preds, target, [], [], num_outputs=1 if preds.ndim == 1 else preds.shape[-1]
    )
    tau, p_value = _kendall_corrcoef_compute(dim_zero_cat(_preds), dim_zero_cat(_target), _variant, _alternative)
    if p_value is not None:
        return tau, p_value
    return tau
