"""Host layer of panoptic quality (reference: functional/detection/_panoptic_quality_common.py): argument and input
validation with the reference's exceptions and messages, the update on kernel K18, and the ``[K]`` epilogue in torch ops.

An update never leaves the device except for one read of K18's error word; the reference validates its inputs on the host
in every update as well."""
from __future__ import annotations

from collections.abc import Collection

import torch
from torch import Tensor

from metrics_b200 import _native
from metrics_b200.utilities.prints import rank_zero_warn

_INTEGER_DTYPES = (torch.int64, torch.int32, torch.int16, torch.int8, torch.uint8)


def _parse_categories(things: Collection[int], stuffs: Collection[int]) -> tuple[set[int], set[int]]:
    """The de-duplicated ``things`` and ``stuffs`` sets; warns on duplicates, raises on non-int, shared or no categories."""
    parsed = []
    for name, values in (("things", things), ("stuffs", stuffs)):
        unique = set(values)
        if len(unique) < len(values):
            rank_zero_warn(f"The provided `{name}` categories contained duplicates, which have been removed.", UserWarning)
        parsed.append(unique)
    things_set, stuffs_set = parsed
    for name, given, unique in (("things", things, things_set), ("stuffs", stuffs, stuffs_set)):
        if any(not isinstance(v, int) for v in unique):
            raise TypeError(f"Expected argument `{name}` to contain `int` categories, but got {given}")
    if things_set & stuffs_set:
        raise ValueError(f"Expected arguments `things` and `stuffs` to have distinct keys, but got {things} and {stuffs}")
    if not things_set | stuffs_set:
        raise ValueError("At least one of `things` and `stuffs` must be non-empty.")
    return things_set, stuffs_set


def _validate_inputs(preds: Tensor, target: Tensor) -> None:
    """Types and shapes: two tensors of one shape ``(B, *spatial_dims, 2)`` with at least one spatial dimension."""
    for name, x in (("preds", preds), ("target", target)):
        if not isinstance(x, Tensor):
            raise TypeError(f"Expected argument `{name}` to be of type `torch.Tensor`, but got {type(x)}")
    if preds.shape != target.shape:
        raise ValueError(
            f"Expected argument `preds` and `target` to have the same shape, but got {preds.shape} and {target.shape}"
        )
    if preds.dim() < 3:
        raise ValueError(
            f"Expected argument `preds` to have at least one spatial dimension (B, *spatial_dims, 2), got {preds.shape}"
        )
    if preds.shape[-1] != 2:
        raise ValueError(
            "Expected argument `preds` to have exactly 2 channels in the last dimension (category, instance), "
            f"got {preds.shape} instead"
        )


def _get_void_color(things: set[int], stuffs: set[int]) -> tuple[int, int]:
    """The color unknown categories become: a category id above every known one, instance 0."""
    return 1 + max([0, *things, *stuffs]), 0


def _get_category_id_to_continuous_id(things: set[int], stuffs: set[int]) -> dict[int, int]:
    """Continuous ids: sorted things ``0 .. len(things) - 1``, then sorted stuffs."""
    order = sorted(things) + sorted(stuffs)
    return {cat: i for i, cat in enumerate(order)}


def _unknown_preds_error(preds: Tensor, things: set[int], stuffs: set[int]) -> ValueError:
    """The reference's error for categories of ``preds`` outside things and stuffs (built on the error path only)."""
    flat = preds.detach().flatten(1, -2)
    known = torch.isin(flat[..., 0], torch.tensor(sorted(things | stuffs), dtype=torch.int64, device=flat.device))
    return ValueError(f"Unknown categories found: {flat[~known]}")


def _check_dtypes(preds: Tensor, target: Tensor) -> None:
    for name, x in (("preds", preds), ("target", target)):
        if x.dtype not in _INTEGER_DTYPES:
            raise ValueError(
                f"Expected argument `{name}` to hold integer (category_id, instance_id) pairs, but got dtype {x.dtype}"
            )


def _panoptic_quality_update(
    preds: Tensor,
    target: Tensor,
    things: set[int],
    stuffs: set[int],
    allow_unknown_preds_category: bool,
    states: tuple[Tensor, Tensor, Tensor, Tensor],
    modified: bool = False,
    categories: Tensor | None = None,
) -> None:
    """Add one batch to ``states = (iou_sum, true_positives, false_positives, false_negatives)`` in place (kernel K18).

    ``modified``: the ModifiedPanopticQuality rule for stuffs.  ``categories``: `_native.panoptic_categories` on the
    inputs' device, built here when None.  Unknown categories in ``preds`` raise ValueError unless
    ``allow_unknown_preds_category``; the states are then unchanged."""
    _check_dtypes(preds, target)
    if categories is None:
        categories = _native.panoptic_categories(things, stuffs, preds.device)
    unknown = _native.panoptic_update_(*states, preds, target, categories, len(things), modified, allow_unknown_preds_category)
    if unknown:
        raise _unknown_preds_error(preds, things, stuffs)


def _panoptic_quality_compute(
    iou_sum: Tensor,
    true_positives: Tensor,
    false_positives: Tensor,
    false_negatives: Tensor,
) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """Per-class ``pq, sq, rq`` and their means over the classes with a non-zero denominator (float64 ``sq`` and ``pq``,
    float32 ``rq``, as the reference promotes them)."""
    sq = torch.where(true_positives > 0.0, iou_sum / true_positives, 0.0)
    denominator = true_positives + 0.5 * false_positives + 0.5 * false_negatives
    rq = torch.where(denominator > 0.0, true_positives / denominator, 0.0)
    pq = sq * rq
    seen = denominator > 0
    return pq, sq, rq, torch.mean(pq[seen]), torch.mean(sq[seen]), torch.mean(rq[seen])


def _panoptic_quality_output(pq: Tensor, sq: Tensor, rq: Tensor, pq_avg: Tensor, sq_avg: Tensor, rq_avg: Tensor,
                             return_sq_and_rq: bool, return_per_class: bool) -> Tensor:
    """A scalar, ``[3]``, ``[1, K]`` or ``[K, 3]`` by the two flags."""
    if return_per_class:
        return torch.stack((pq, sq, rq), dim=-1) if return_sq_and_rq else pq.view(1, -1)
    return torch.stack((pq_avg, sq_avg, rq_avg), dim=0) if return_sq_and_rq else pq_avg


def _zero_states(num_categories: int, device) -> tuple[Tensor, Tensor, Tensor, Tensor]:
    iou_sum = torch.zeros(num_categories, dtype=torch.double, device=device)
    counts = [torch.zeros(num_categories, dtype=torch.int, device=device) for _ in range(3)]
    return iou_sum, counts[0], counts[1], counts[2]
