"""Operating-point metrics read off a curve: recall@precision, precision@recall, sensitivity@specificity,
specificity@sensitivity (binary / multiclass / multilabel, exact and binned).

Reference: functional/classification/{recall_fixed_precision,precision_fixed_recall,sensitivity_specificity,
specificity_sensitivity}.py.  The curves come from the sort + scan kernels (exact) or the K4 state (binned); the
selection of the operating point is a lexicographic arg-max over the curve points, done here with masked device
reductions (no Python loop over thresholds, no host sync) — SURVEY.md §8(f) row 3.
"""
from __future__ import annotations

from typing import Callable, Dict, List, NamedTuple, Optional, Sequence, Union

import torch
from torch import Tensor
from typing_extensions import Literal

from metrics_b200.functional.classification.precision_recall_curve import (
    _binary_precision_recall_curve_arg_validation,
    _binary_precision_recall_curve_compute,
    _binary_precision_recall_curve_format,
    _binary_precision_recall_curve_tensor_validation,
    _binary_precision_recall_curve_update,
    _multiclass_precision_recall_curve_arg_validation,
    _multiclass_precision_recall_curve_compute,
    _multiclass_precision_recall_curve_format,
    _multiclass_precision_recall_curve_tensor_validation,
    _multiclass_precision_recall_curve_update,
    _multilabel_precision_recall_curve_arg_validation,
    _multilabel_precision_recall_curve_compute,
    _multilabel_precision_recall_curve_format,
    _multilabel_precision_recall_curve_tensor_validation,
    _multilabel_precision_recall_curve_update,
)
from metrics_b200.functional.classification.roc import _binary_roc_compute, _multiclass_roc_compute, _multilabel_roc_compute


def _first_lex_max(keys: Sequence[Tensor], mask: Tensor) -> Tensor:
    """Index of the lexicographically largest row of ``zip(*keys)`` among ``mask`` (first one among full ties)."""
    live = mask
    for key in keys:
        neg = torch.full_like(key, float("-inf"))
        best = torch.where(live, key, neg).max()
        live = live & (key == best)
    return torch.argmax(live.to(torch.uint8))


def _recall_at_precision(precision: Tensor, recall: Tensor, thresholds: Tensor, min_precision: float):
    """Highest recall with precision >= min_precision; ties -> higher precision, then higher threshold
    (reference recall_fixed_precision.py:58-77: `_lexargmax` over (recall, precision, threshold))."""
    n = min(recall.shape[0], precision.shape[0], thresholds.shape[0])
    p, r, t = precision[:n], recall[:n], thresholds[:n]
    mask = p >= min_precision
    idx = _first_lex_max((r, p, t), mask)
    found = mask.any()
    value = torch.where(found, r[idx], torch.zeros((), dtype=r.dtype, device=r.device))
    big = torch.full((), 1e6, dtype=t.dtype, device=t.device)
    return value, torch.where(found & (value != 0), t[idx], big)


def _precision_at_recall(precision: Tensor, recall: Tensor, thresholds: Tensor, min_recall: float):
    """Highest precision with recall >= min_recall; ties -> higher recall, then higher threshold (reference
    precision_fixed_recall.py:42-60: Python `max` over (precision, recall, threshold) tuples)."""
    n = min(recall.shape[0], precision.shape[0], thresholds.shape[0])
    p, r, t = precision[:n], recall[:n], thresholds[:n]
    mask = r >= min_recall
    idx = _first_lex_max((p, r, t), mask)
    found = mask.any()
    value = torch.where(found, p[idx], torch.zeros((), dtype=p.dtype, device=p.device))
    big = torch.full((), 1e6, dtype=t.dtype, device=t.device)
    return value, torch.where(found & (value != 0), t[idx], big)


def _best_with_floor(objective: Tensor, constraint: Tensor, thresholds: Tensor, floor: float):
    """First arg-max of ``objective`` among the points with ``constraint >= floor`` (0 / 1e6 if there is none) —
    reference sensitivity_specificity.py:47-70 and specificity_sensitivity.py:48-71."""
    mask = constraint >= floor
    idx = torch.argmax(torch.where(mask, objective, torch.full_like(objective, float("-inf"))))
    found = mask.any()
    value = torch.where(found, objective[idx], torch.zeros((), dtype=objective.dtype, device=objective.device))
    big = torch.full((), 1e6, dtype=thresholds.dtype, device=thresholds.device)
    return value, torch.where(found, thresholds[idx], big)


class _Family(NamedTuple):
    arg: str  # name of the floor argument
    curve: str  # "prc" | "roc"
    pick: Callable  # (curve_a, curve_b, thresholds, floor) -> (value, threshold)
    reference: str


def _convert_fpr_to_specificity(fpr: Tensor) -> Tensor:
    """Specificity is the complement of the false-positive rate (reference sensitivity_specificity.py:42-44)."""
    return 1 - fpr


def _pick_sens_at_spec(fpr: Tensor, tpr: Tensor, thresholds: Tensor, floor: float):
    return _best_with_floor(tpr, _convert_fpr_to_specificity(fpr), thresholds, floor)


def _pick_spec_at_sens(fpr: Tensor, tpr: Tensor, thresholds: Tensor, floor: float):
    return _best_with_floor(_convert_fpr_to_specificity(fpr), tpr, thresholds, floor)


_FAMILIES: Dict[str, _Family] = {
    "recall_at_fixed_precision": _Family("min_precision", "prc", _recall_at_precision, "recall_fixed_precision.py"),
    "precision_at_fixed_recall": _Family("min_recall", "prc", _precision_at_recall, "precision_fixed_recall.py"),
    "sensitivity_at_specificity": _Family("min_specificity", "roc", _pick_sens_at_spec, "sensitivity_specificity.py"),
    "specificity_at_sensitivity": _Family("min_sensitivity", "roc", _pick_spec_at_sens, "specificity_sensitivity.py"),
}


def _floor_validation(name: str, value: float) -> None:
    if not isinstance(value, float) and not (0 <= value <= 1):
        raise ValueError(f"Expected argument `{name}` to be an float in the [0,1] range, but got {value}")


def _named_floor(fam: _Family, floor: Optional[float], named: dict) -> float:
    """The reference names the floor argument per family (`min_precision`, `min_recall`, ...): accept it by keyword too."""
    if floor is None:
        if set(named) != {fam.arg}:
            raise TypeError(f"expected the keyword argument `{fam.arg}`, got {sorted(named)}")
        return named[fam.arg]
    if named:
        raise TypeError(f"unexpected keyword arguments {sorted(named)}")
    return floor


def _per_curve(fam: _Family, a: Union[Tensor, List[Tensor]], b: Union[Tensor, List[Tensor]],
               thresholds: Union[Tensor, List[Tensor]], floor: float, shared_thresholds: bool):
    res = [fam.pick(x, y, thresholds if shared_thresholds else thresholds[i], floor) for i, (x, y) in enumerate(zip(a, b))]
    return torch.stack([r[0] for r in res]), torch.stack([r[1] for r in res])


def _binary_at_fixed_compute(kind: str, state, thresholds: Optional[Tensor], floor: float, pos_label: int = 1):
    fam = _FAMILIES[kind]
    if fam.curve == "prc":
        a, b, t = _binary_precision_recall_curve_compute(state, thresholds, pos_label)
    else:
        a, b, t = _binary_roc_compute(state, thresholds, pos_label)
    return fam.pick(a, b, t, floor)


def _multiclass_at_fixed_compute(kind: str, state, num_classes: int, thresholds: Optional[Tensor], floor: float):
    fam = _FAMILIES[kind]
    if fam.curve == "prc":
        a, b, t = _multiclass_precision_recall_curve_compute(state, num_classes, thresholds)
    else:
        a, b, t = _multiclass_roc_compute(state, num_classes, thresholds)
    return _per_curve(fam, a, b, t, floor, isinstance(state, Tensor))


def _multilabel_at_fixed_compute(kind: str, state, num_labels: int, thresholds: Optional[Tensor],
                                 ignore_index: Optional[int], floor: float):
    fam = _FAMILIES[kind]
    if fam.curve == "prc":
        a, b, t = _multilabel_precision_recall_curve_compute(state, num_labels, thresholds, ignore_index)
    else:
        a, b, t = _multilabel_roc_compute(state, num_labels, thresholds, ignore_index)
    return _per_curve(fam, a, b, t, floor, isinstance(state, Tensor))


def _publish_signature(fn: Callable, arg: str) -> Callable:
    """Introspection parity: present the shared `floor` parameter under the family's own name (`min_precision`, ...), as a
    required argument and without the catch-all that implements it, so `inspect.signature` shows the reference's signature."""
    import inspect

    params = []
    for prm in inspect.signature(fn).parameters.values():
        if prm.name == "floor":
            params.append(prm.replace(name=arg, default=inspect.Parameter.empty, annotation=float))
        elif prm.kind is inspect.Parameter.VAR_KEYWORD and prm.name == "named":
            continue
        else:
            params.append(prm)
    fn.__signature__ = inspect.Signature(params)
    return fn


def _make_binary(kind: str) -> Callable:
    fam = _FAMILIES[kind]

    def fn_(preds: Tensor, target: Tensor, floor: Optional[float] = None,
            thresholds: Optional[Union[int, List[float], Tensor]] = None, ignore_index: Optional[int] = None,
            validate_args: bool = True, **named: float):
        floor = _named_floor(fam, floor, named)
        if validate_args:
            _binary_precision_recall_curve_arg_validation(thresholds, ignore_index)
            _floor_validation(fam.arg, floor)
            _binary_precision_recall_curve_tensor_validation(preds, target, ignore_index)
        preds, target, thresholds = _binary_precision_recall_curve_format(preds, target, thresholds, ignore_index)
        state = _binary_precision_recall_curve_update(preds, target, thresholds)
        return _binary_at_fixed_compute(kind, state, thresholds, floor)

    fn_.__name__ = fn_.__qualname__ = f"binary_{kind}"
    fn_.__doc__ = f"Binary {kind.replace('_', ' ')} (reference functional/classification/{fam.reference}); `floor` = `{fam.arg}`."
    return _publish_signature(fn_, fam.arg)


def _make_multiclass(kind: str) -> Callable:
    fam = _FAMILIES[kind]

    def fn_(preds: Tensor, target: Tensor, num_classes: int, floor: Optional[float] = None,
            thresholds: Optional[Union[int, List[float], Tensor]] = None, ignore_index: Optional[int] = None,
            validate_args: bool = True, **named: float):
        floor = _named_floor(fam, floor, named)
        if validate_args:
            _multiclass_precision_recall_curve_arg_validation(num_classes, thresholds, ignore_index)
            _floor_validation(fam.arg, floor)
            _multiclass_precision_recall_curve_tensor_validation(preds, target, num_classes, ignore_index)
        preds, target, thresholds = _multiclass_precision_recall_curve_format(preds, target, num_classes, thresholds, ignore_index)
        state = _multiclass_precision_recall_curve_update(preds, target, num_classes, thresholds)
        return _multiclass_at_fixed_compute(kind, state, num_classes, thresholds, floor)

    fn_.__name__ = fn_.__qualname__ = f"multiclass_{kind}"
    fn_.__doc__ = f"Multiclass one-vs-rest {kind.replace('_', ' ')} (reference {fam.reference}); `floor` = `{fam.arg}`."
    return _publish_signature(fn_, fam.arg)


def _make_multilabel(kind: str) -> Callable:
    fam = _FAMILIES[kind]

    def fn_(preds: Tensor, target: Tensor, num_labels: int, floor: Optional[float] = None,
            thresholds: Optional[Union[int, List[float], Tensor]] = None, ignore_index: Optional[int] = None,
            validate_args: bool = True, **named: float):
        floor = _named_floor(fam, floor, named)
        if validate_args:
            _multilabel_precision_recall_curve_arg_validation(num_labels, thresholds, ignore_index)
            _floor_validation(fam.arg, floor)
            _multilabel_precision_recall_curve_tensor_validation(preds, target, num_labels, ignore_index)
        preds, target, thresholds = _multilabel_precision_recall_curve_format(preds, target, num_labels, thresholds, ignore_index)
        state = _multilabel_precision_recall_curve_update(preds, target, num_labels, thresholds, ignore_index)
        return _multilabel_at_fixed_compute(kind, state, num_labels, thresholds, ignore_index, floor)

    fn_.__name__ = fn_.__qualname__ = f"multilabel_{kind}"
    fn_.__doc__ = f"Multilabel per-label {kind.replace('_', ' ')} (reference {fam.reference}); `floor` = `{fam.arg}`."
    return _publish_signature(fn_, fam.arg)


binary_recall_at_fixed_precision = _make_binary("recall_at_fixed_precision")
multiclass_recall_at_fixed_precision = _make_multiclass("recall_at_fixed_precision")
multilabel_recall_at_fixed_precision = _make_multilabel("recall_at_fixed_precision")
binary_precision_at_fixed_recall = _make_binary("precision_at_fixed_recall")
multiclass_precision_at_fixed_recall = _make_multiclass("precision_at_fixed_recall")
multilabel_precision_at_fixed_recall = _make_multilabel("precision_at_fixed_recall")
binary_sensitivity_at_specificity = _make_binary("sensitivity_at_specificity")
multiclass_sensitivity_at_specificity = _make_multiclass("sensitivity_at_specificity")
multilabel_sensitivity_at_specificity = _make_multilabel("sensitivity_at_specificity")
binary_specificity_at_sensitivity = _make_binary("specificity_at_sensitivity")
multiclass_specificity_at_sensitivity = _make_multiclass("specificity_at_sensitivity")
multilabel_specificity_at_sensitivity = _make_multilabel("specificity_at_sensitivity")


def _make_task(kind: str, b: Callable, mc: Callable, ml: Callable) -> Callable:
    fam = _FAMILIES[kind]

    def fn_(preds: Tensor, target: Tensor, task: Literal["binary", "multiclass", "multilabel"], floor: Optional[float] = None,
            thresholds: Optional[Union[int, List[float], Tensor]] = None, num_classes: Optional[int] = None,
            num_labels: Optional[int] = None, ignore_index: Optional[int] = None, validate_args: bool = True,
            **named: float):
        from metrics_b200.functional.classification._task import call_for_task

        floor = _named_floor(fam, floor, named)
        return call_for_task(task, num_classes, num_labels,
                             lambda: b(preds, target, floor, thresholds, ignore_index, validate_args),
                             lambda c: mc(preds, target, c, floor, thresholds, ignore_index, validate_args),
                             lambda n: ml(preds, target, n, floor, thresholds, ignore_index, validate_args))

    fn_.__name__ = fn_.__qualname__ = kind
    fn_.__doc__ = f"Task wrapper for {kind.replace('_', ' ')} (reference {fam.reference}); `floor` = `{fam.arg}`."
    return _publish_signature(fn_, fam.arg)


recall_at_fixed_precision = _make_task("recall_at_fixed_precision", binary_recall_at_fixed_precision,
                                       multiclass_recall_at_fixed_precision, multilabel_recall_at_fixed_precision)
precision_at_fixed_recall = _make_task("precision_at_fixed_recall", binary_precision_at_fixed_recall,
                                       multiclass_precision_at_fixed_recall, multilabel_precision_at_fixed_recall)
sensitivity_at_specificity = _make_task("sensitivity_at_specificity", binary_sensitivity_at_specificity,
                                        multiclass_sensitivity_at_specificity, multilabel_sensitivity_at_specificity)
specificity_at_sensitivity = _make_task("specificity_at_sensitivity", binary_specificity_at_sensitivity,
                                        multiclass_specificity_at_sensitivity, multilabel_specificity_at_sensitivity)
