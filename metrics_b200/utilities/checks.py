"""Shape checks shared by the functional front-ends (reference: utilities/checks.py:38-43)."""
from torch import Tensor


def _check_same_shape(preds: Tensor, target: Tensor) -> None:
    if preds.shape != target.shape:
        raise RuntimeError(
            f"Predictions and targets are expected to have the same shape, but got {preds.shape} and {target.shape}."
        )


def _allclose_recursive(res1, res2, atol: float = 1e-6) -> bool:
    """Structural comparison of two metric results (tensors within ``atol``, containers element-wise) — reference
    utilities/checks.py:620-631."""
    from collections.abc import Mapping, Sequence

    import torch

    if isinstance(res1, Tensor):
        return bool(torch.allclose(res1, res2, atol=atol))
    if isinstance(res1, str):
        return res1 == res2
    if isinstance(res1, Mapping):
        return all(_allclose_recursive(res1[key], res2[key], atol) for key in res1)
    if isinstance(res1, Sequence):
        return all(_allclose_recursive(a, b, atol) for a, b in zip(res1, res2))
    return res1 == res2


def _unwrapped(fn):
    """Peel `functools.wraps` layers, `Mock(wraps=...)` and `functools.partial` off a callable."""
    from functools import partial
    from unittest.mock import Mock

    for _ in range(16):
        if fn is None:
            break
        if hasattr(fn, "__wrapped__"):
            fn = fn.__wrapped__
        elif isinstance(fn, Mock):
            fn = fn._mock_wraps
        elif isinstance(fn, partial):
            fn = fn.func
        else:
            break
    return fn


def is_overridden(method_name: str, instance: object, parent: object) -> bool:
    """Whether ``instance`` provides its own ``method_name`` rather than ``parent``'s (reference checks.py:740-762);
    decorated, mocked and partial-bound methods are compared by the function underneath."""
    own = _unwrapped(getattr(instance, method_name, None))
    if own is None:
        return False
    inherited = getattr(parent, method_name, None)
    if inherited is None:
        raise ValueError("The parent should define the method")
    return own.__code__ is not inherited.__code__


def check_forward_full_state_property(metric_class, init_args=None, input_args=None, num_update_to_compare=[10, 100, 1000],  # noqa: B006 (read only; the reference's default)
                                      reps: int = 5) -> None:
    """Tell whether ``full_state_update = False`` is safe for ``metric_class`` and whether it is faster
    (reference checks.py:635-737): run ``forward`` both ways on the same inputs, compare every batch value and the final
    ``compute()``; when they agree, time both and print the recommendation in the reference's wording."""
    from time import perf_counter

    import torch

    init_args, input_args = init_args or {}, input_args or {}
    variants = [type(name, (metric_class,), {"full_state_update": flag})(**init_args)
                for name, flag in (("FullState", True), ("PartState", False))]
    full, part = variants
    same = True
    try:  # an exception in the reduced-state path means `update` needs the accumulated state
        for _ in range(num_update_to_compare[0]):
            same = same and _allclose_recursive(full(**input_args), part(**input_args))
        same = same and _allclose_recursive(full.compute(), part.compute())
    except RuntimeError:
        same = False
    if not same:
        print("Recommended setting `full_state_update=True`")
        return
    seconds = torch.zeros(2, len(num_update_to_compare), reps)
    for i, metric in enumerate(variants):
        for j, steps in enumerate(num_update_to_compare):
            for r in range(reps):
                start = perf_counter()
                for _ in range(steps):
                    metric(**input_args)
                seconds[i, j, r] = perf_counter() - start
                metric.reset()
    mean, std = seconds.mean(-1), seconds.std(-1)
    for j, steps in enumerate(num_update_to_compare):
        print(f"Full state for {steps} steps took: {mean[0, j]}+-{std[0, j]:0.3f}")
        print(f"Partial state for {steps} steps took: {mean[1, j]:0.3f}+-{std[1, j]:0.3f}")
    print(f"Recommended setting `full_state_update={not bool(mean[1, -1] < mean[0, -1])}`")


def _check_retrieval_functional_inputs(preds: Tensor, target: Tensor, allow_non_binary_target: bool = False):
    """``(preds float32, target int64 or float32)``, flattened, of one query (reference checks.py:508-536): same shape,
    non-empty, then `_check_retrieval_target_and_prediction_types`."""
    if preds.shape != target.shape:
        raise ValueError("`preds` and `target` must be of the same shape")
    if not preds.numel() or not preds.size():
        raise ValueError("`preds` and `target` must be non-empty and non-scalar tensors")
    return _check_retrieval_target_and_prediction_types(preds, target, allow_non_binary_target=allow_non_binary_target)


def _check_retrieval_inputs(indexes: Tensor, preds: Tensor, target: Tensor, allow_non_binary_target: bool = False,
                            ignore_index=None):
    """``(indexes int64, preds float32, target)`` flattened, with the records whose target is ``ignore_index`` removed
    (reference checks.py:539-585).  The ``ignore_index`` mask and the binary-target check read values on the host."""
    import torch

    if indexes.shape != preds.shape or preds.shape != target.shape:
        raise ValueError("`indexes`, `preds` and `target` must be of the same shape")
    if indexes.dtype is not torch.long:
        raise ValueError("`indexes` must be a tensor of long integers")
    if ignore_index is not None:
        keep = target != ignore_index
        indexes, preds, target = indexes[keep], preds[keep], target[keep]
    if not indexes.numel() or not indexes.size():
        raise ValueError("`indexes`, `preds` and `target` must be non-empty and non-scalar tensors")
    preds, target = _check_retrieval_target_and_prediction_types(preds, target, allow_non_binary_target=allow_non_binary_target)
    return indexes.long().flatten(), preds, target


def _check_retrieval_target_and_prediction_types(preds: Tensor, target: Tensor, allow_non_binary_target: bool = False):
    """Dtype checks of a retrieval batch (reference checks.py:588-615): bool / int32 / int64 / floating targets, floating
    scores, binary targets unless ``allow_non_binary_target``.  Returns flat ``preds`` float32 and ``target`` float32 when
    floating, else int64."""
    import torch

    if target.dtype not in (torch.bool, torch.long, torch.int) and not torch.is_floating_point(target):
        raise ValueError("`target` must be a tensor of booleans, integers or floats")
    if not preds.is_floating_point():
        raise ValueError("`preds` must be a tensor of floats")
    if not allow_non_binary_target and (target.max() > 1 or target.min() < 0):
        raise ValueError("`target` must contain `binary` values")
    target = target.float() if target.is_floating_point() else target.long()
    return preds.float().flatten(), target.flatten()
