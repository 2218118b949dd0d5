"""Shared panoptic-quality cases: built from fixed seeds, so the golden maker (run against the reference) and the tests
(run against this package) see the same inputs.  Each case is a dict:

    name, modified (ModifiedPanopticQuality), things, stuffs, kwargs (constructor / functional flags), batches [(preds,
    target), ...] of integer tensors [B, *spatial, 2].

`golden_cases()` are the ones the reference evaluates (small enough for its per-pair Python loop); `oracle_only_cases()`
are checked against the oracle alone."""
from __future__ import annotations

import torch

# the reference's unit-test inputs (one image each, repeated as two batches)
_P0 = [[[6, 0], [0, 0], [6, 0], [6, 0], [0, 1]], [[0, 0], [0, 0], [6, 0], [0, 1], [0, 1]],
       [[0, 0], [0, 0], [6, 0], [0, 1], [1, 0]], [[0, 0], [7, 0], [6, 0], [1, 0], [1, 0]],
       [[0, 0], [7, 0], [7, 0], [7, 0], [7, 0]]]
_T0 = [[[6, 0], [6, 0], [6, 0], [6, 0], [0, 0]], [[0, 1], [0, 1], [6, 0], [0, 0], [0, 0]],
       [[0, 1], [0, 1], [6, 0], [1, 0], [1, 0]], [[0, 1], [7, 0], [7, 0], [1, 0], [1, 0]],
       [[0, 1], [7, 0], [7, 0], [7, 0], [7, 0]]]
_P1 = [[10, 0], [10, 123], [0, 1], [10, 0], [1, 2]]
_T1 = [[10, 0], [10, 0], [0, 0], [0, 1], [1, 0]]
ARGS = ({"things": {0, 1}, "stuffs": {6, 7}}, {"things": {2}, "stuffs": {3}, "allow_unknown_preds_category": True},
        {"things": {0, 1}, "stuffs": {10, 11}})
# the docstring examples
_DOC_P = [[[6, 0], [0, 0], [6, 0], [6, 0]], [[0, 0], [0, 0], [6, 0], [0, 1]], [[0, 0], [0, 0], [6, 0], [0, 1]],
          [[0, 0], [7, 0], [6, 0], [1, 0]], [[0, 0], [7, 0], [7, 0], [7, 0]]]
_DOC_T = [[[6, 0], [0, 1], [6, 0], [0, 1]], [[0, 1], [0, 1], [6, 0], [0, 1]], [[0, 1], [0, 1], [6, 0], [1, 0]],
          [[0, 1], [7, 0], [1, 0], [1, 0]], [[0, 1], [7, 0], [7, 0], [7, 0]]]
INT_DTYPES = (torch.int64, torch.int32, torch.int16, torch.int8, torch.uint8)
FLAGS = ({}, {"return_sq_and_rq": True}, {"return_per_class": True}, {"return_sq_and_rq": True, "return_per_class": True})


def inputs0():
    return torch.tensor(_P0)[None], torch.tensor(_T0)[None]


def inputs1():
    return torch.tensor(_P1)[None], torch.tensor(_T1)[None]


def _case(name, modified, things, stuffs, batches, **kwargs):
    return {"name": name, "modified": modified, "things": set(things), "stuffs": set(stuffs), "kwargs": kwargs,
            "batches": batches}


def blocky(g, shape, cats, n_inst, block=4, dtype=torch.int64, inst_lo=0):
    """[B, *spatial, 2] maps of constant (category, instance) blocks along the last spatial axis."""
    b, *sp = shape
    small = [*sp[:-1], (sp[-1] + block - 1) // block]
    cat = torch.tensor(cats)[torch.randint(0, len(cats), (b, *small), generator=g)]
    inst = torch.randint(inst_lo, inst_lo + n_inst, (b, *small), generator=g)
    x = torch.stack([cat, inst], -1).repeat_interleave(block, -2)[..., : sp[-1], :]
    return x.to(dtype).contiguous()


def perturb(g, x, frac, cats, n_inst):
    """`x` with a fraction of its points relabelled."""
    y = x.clone()
    m = torch.rand(x.shape[:-1], generator=g) < frac
    y[..., 0][m] = torch.tensor(cats, dtype=x.dtype)[torch.randint(0, len(cats), (int(m.sum()),), generator=g)]
    y[..., 1][m] = torch.randint(0, n_inst, (int(m.sum()),), generator=g).to(x.dtype)
    return y


def golden_cases() -> list:
    g = torch.Generator().manual_seed(1818)
    out = []
    i0, i1 = inputs0(), inputs1()
    for mod in (False, True):
        tag = "mpq" if mod else "pq"
        for ii, ai in ((0, 0), (0, 1), (1, 2)):  # the combinations the reference tests (the others hold unknown preds)
            args = ARGS[ai]
            kw = {k: v for k, v in args.items() if k not in ("things", "stuffs")}
            out.append(_case(f"{tag}_inputs{ii}_args{ai}", mod, args["things"], args["stuffs"], [(i0, i1)[ii]] * 2, **kw))
        # class order: (class type, ids)
        for kind, ids in (("stuffs", (0, 2, 1)), ("stuffs", (0, 3, 2)), ("stuffs", (0, 10, 2)), ("things", (0, 2, 1)),
                          ("things", (0, 3, 2)), ("things", (0, 10, 2))):
            a, b, c = ([x, 0] for x in ids)
            p, t = torch.tensor([a, a, b, b, b, c])[None], torch.tensor([a, a, b, b, c, c])[None]
            things, stuffs = (ids, ()) if kind == "things" else ((), ids)
            kw = {} if mod else {"return_per_class": True}
            out.append(_case(f"{tag}_order_{kind}_{'_'.join(map(str, ids))}", mod, things, stuffs, [(p, t), (p, t)], **kw))
        # extreme values
        t = i0[1]
        out.append(_case(f"{tag}_identity", mod, {0, 1}, {6, 7}, [(t, t)]))
        out.append(_case(f"{tag}_shifted", mod, {0, 1}, {6, 7}, [(t, t + 1)]))
        # ignore masks: an unknown-category block appended to the target along each axis
        for ii, (inp, args) in enumerate(((i0, ARGS[0]), (i1, ARGS[2]))):
            p, t = inp
            for dim in range(p.dim() - 1):
                ign = torch.zeros_like(p)
                ign[..., 0] = 255
                out.append(_case(f"{tag}_ignore{ii}_dim{dim}", mod, args["things"], args["stuffs"],
                                 [(torch.cat([p, p], dim), torch.cat([t, ign], dim))]))
        # docstring examples
        dp, dt = torch.tensor(_DOC_P)[None], torch.tensor(_DOC_T)[None]
        for fi, flags in enumerate(FLAGS if not mod else ({},)):
            out.append(_case(f"{tag}_doc{fi}", mod, {0, 1}, {6, 7}, [(dp, dt)], **flags))
        mp = torch.tensor([[[0, 0], [0, 1], [6, 0], [7, 0], [0, 2], [1, 0]]])
        mt = torch.tensor([[[0, 1], [0, 0], [6, 0], [7, 0], [6, 0], [255, 0]]])
        out.append(_case(f"{tag}_doc_modified", mod, {0, 1}, {6, 7}, [(mp, mt)]))
        # seeded blocky maps in every integer dtype; stuff points keep non-zero instance ids; categories 0 and 9 unknown
        cats = [0, 1, 2, 3, 4, 5, 6, 9]
        for di, dtype in enumerate(INT_DTYPES):
            for fi, flags in enumerate(FLAGS if not mod else ({},)):
                batches = []
                for _ in range(2):
                    t = blocky(g, (3, 12, 16), cats, 3, dtype=dtype)
                    p = perturb(g, t, 0.2, cats[1:-1], 3)
                    batches.append((p, t))
                out.append(_case(f"{tag}_blocky_{str(dtype)[6:]}_{fi}", mod, {1, 2, 3}, {4, 5, 6}, batches,
                                 allow_unknown_preds_category=True, **flags))
        # point clouds [B, N, 2] and volumes [B, D, H, W, 2]
        t = blocky(g, (2, 64), [1, 2, 5, 6], 4, block=8)
        out.append(_case(f"{tag}_points", mod, {1, 2}, {5, 6}, [(perturb(g, t, 0.25, [1, 2, 5, 6], 4), t)]))
        t = blocky(g, (2, 3, 6, 8), [1, 2, 5, 6], 3, block=4)
        out.append(_case(f"{tag}_volume", mod, {1, 2}, {5, 6}, [(perturb(g, t, 0.25, [1, 2, 5, 6], 3), t)]))
        # negative instance ids and ids >= 2^40 (int64)
        t = blocky(g, (2, 10, 12), [1, 2, 5], 3, inst_lo=-1)
        t[..., 1] = torch.where(t[..., 1] > 0, t[..., 1] + (1 << 40), t[..., 1])
        p = perturb(g, t, 0.15, [1, 2, 5], 2)
        p[..., 1] = torch.where(p[..., 1] == 1, torch.full_like(p[..., 1], (1 << 40) + 1), p[..., 1])
        out.append(_case(f"{tag}_wide_instances", mod, {1, 2}, {5}, [(p, t)]))
        # IoU exactly 0.5 (inter 2, union 4: no match) and a pred segment exactly half void (a false positive)
        p = torch.tensor([[[1, 1], [1, 1], [1, 1], [2, 0], [5, 0], [5, 0], [5, 0], [5, 0]]])
        t = torch.tensor([[[2, 0], [1, 1], [1, 1], [1, 1], [8, 0], [8, 0], [5, 0], [5, 0]]])
        out.append(_case(f"{tag}_half", mod, {1, 2}, {5}, [(p, t)]))
        # unknown categories in target and, with the flag set, in preds
        t = blocky(g, (2, 8, 8), [1, 2, 5, 7, 8], 2)
        p = perturb(g, t, 0.3, [1, 2, 3, 5, 7], 2)
        out.append(_case(f"{tag}_unknown", mod, {1, 2}, {5, 7}, [(p, t)], allow_unknown_preds_category=True))
        # an empty batch
        e = torch.zeros(0, 4, 4, 2, dtype=torch.int64)
        out.append(_case(f"{tag}_empty_batch", mod, {1}, {2}, [(e, e)]))
    return out


def oracle_only_cases() -> list:
    """A 4097 x 4097 frame with areas above 2^24, where rounding the operands to float32 decides a false negative: target
    segment (1, 1) has 2^24 + 3 points, 2^23 + 2 of them void in preds, so float32(2^23 + 2) / float32(2^24 + 3) is exactly
    0.5 (counted) while the exact ratio is above 0.5 (not counted).  The rest of the segment is split over three pred
    segments, none of which matches it."""
    side = 4097
    n = side * side
    a = (1 << 24) + 3
    t = torch.zeros(n, 2, dtype=torch.int32)
    t[:, 0] = 5
    t[:a] = torch.tensor([1, 1], dtype=torch.int32)
    p = t.clone()
    v = (1 << 23) + 2
    p[:v] = torch.tensor([9, 0], dtype=torch.int32)  # unknown category: void
    rest = torch.arange(a - v, dtype=torch.int32)
    p[v:a, 1] = 7 + rest * 3 // (a - v)
    p, t = p.view(1, side, side, 2), t.view(1, side, side, 2)
    return [_case("big_areas", False, {1}, {5}, [(p, t)], allow_unknown_preds_category=True),
            _case("big_areas_mpq", True, {1}, {5}, [(p, t)], allow_unknown_preds_category=True)]


STATES = ("iou_sum", "true_positives", "false_positives", "false_negatives")


def load():
    import os

    import numpy as np

    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "panoptic.npz"), allow_pickle=False)


def assert_states(golden, name, got):
    """``got``: the four states (tensors or arrays), bit-equal to the reference's."""
    import numpy as np

    for s, g in zip(STATES, got):
        g = g.cpu().numpy() if hasattr(g, "cpu") else np.asarray(g)
        want = golden[f"{name}/{s}"]
        assert g.dtype == want.dtype and np.array_equal(g.view(np.uint8), want.view(np.uint8)), (name, s, g, want)


def assert_output(want, got):
    """Outputs equal to the reference's, NaN where it has NaN.  The states are bit-equal; the class means are `torch.mean`
    over at most K values on the states' device, whose summation order differs between CPU and CUDA, so a few float32 ulp
    (the `rq` average) or float64 ulp are allowed."""
    import numpy as np

    got = got.cpu().numpy()
    assert got.dtype == want.dtype and got.shape == want.shape, (got, want)
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=0, equal_nan=True)
