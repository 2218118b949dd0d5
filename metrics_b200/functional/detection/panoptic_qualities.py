"""Panoptic quality and modified panoptic quality, functional (reference: functional/detection/panoptic_qualities.py).

The segment areas and pair intersections of every image come from one read of the inputs (kernel K18)."""
from __future__ import annotations

from collections.abc import Collection

from torch import Tensor

from metrics_b200.functional.detection._panoptic_quality_common import (
    _panoptic_quality_compute,
    _panoptic_quality_output,
    _panoptic_quality_update,
    _parse_categories,
    _validate_inputs,
    _zero_states,
)


def panoptic_quality(
    preds: Tensor,
    target: Tensor,
    things: Collection[int],
    stuffs: Collection[int],
    allow_unknown_preds_category: bool = False,
    return_sq_and_rq: bool = False,
    return_per_class: bool = False,
) -> Tensor:
    r"""`Panoptic Quality`_ :math:`PQ = \frac{IOU}{TP + 0.5 FP + 0.5 FN}` of panoptic segmentations.

    ``preds`` / ``target``: integer CUDA tensors ``(B, *spatial_dims, 2)`` of ``(category_id, instance_id)`` pairs; the
    instance id of a stuff is ignored, and target points of an unknown category are left out.  Unknown categories in
    ``preds`` raise ValueError unless ``allow_unknown_preds_category``.  Returns the class average (float64 scalar),
    ``[pq, sq, rq]`` with ``return_sq_and_rq``, ``[1, K]`` with ``return_per_class`` or ``[K, 3]`` with both; classes are
    the sorted things, then the sorted stuffs."""
    things, stuffs = _parse_categories(things, stuffs)
    _validate_inputs(preds, target)
    states = _zero_states(len(things) + len(stuffs), preds.device)
    _panoptic_quality_update(preds, target, things, stuffs, allow_unknown_preds_category, states)
    return _panoptic_quality_output(*_panoptic_quality_compute(*states), return_sq_and_rq, return_per_class)


def modified_panoptic_quality(
    preds: Tensor,
    target: Tensor,
    things: Collection[int],
    stuffs: Collection[int],
    allow_unknown_preds_category: bool = False,
) -> Tensor:
    r"""`Modified Panoptic Quality`_: panoptic quality where a stuff class scores :math:`\frac{IOU_c}{|S_c|}`, the IoU sum
    of its overlapping segments over its number of target segments.  Inputs as in `panoptic_quality`; returns the class
    average (float64 scalar)."""
    things, stuffs = _parse_categories(things, stuffs)
    _validate_inputs(preds, target)
    states = _zero_states(len(things) + len(stuffs), preds.device)
    _panoptic_quality_update(preds, target, things, stuffs, allow_unknown_preds_category, states, modified=True)
    pq_avg = _panoptic_quality_compute(*states)[3]
    return pq_avg
