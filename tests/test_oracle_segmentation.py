"""CPU: the segmentation oracles (oracle/segmentation.py) against the reference's goldens (tests/golden/segmentation.npz).

The op chain on CPU tensors reproduces the reference's states, `compute()` and functional results bit for bit; the numpy
counts equal the chain's counts exactly; the float64 epilogues agree with the reference within float32 rounding."""
import numpy as np
import pytest
import torch

from oracle import segmentation as osg
from tests import segmentation_cases as sc


@pytest.fixture(scope="module")
def golden():
    return sc.load()


def _chain_states(c, golden, key):
    """The reference class's update loop, restated with the oracle chain."""
    kind, opt, kw = c["kind"], c["option"], dict(num_classes=c["num_classes"], include_background=c["include_background"],
                                                   index=c["index"])
    if kind == 1:
        parts = [osg.dice_update_chain(p, t, **kw) for p, t in c["batches"]]
        return {n: torch.cat([q[i] for q in parts]) for i, n in enumerate(("numerator", "denominator", "support"))}
    score = torch.zeros(golden[f"{key}/score"].shape)
    for p, t in c["batches"]:
        if kind == 0:
            s = osg.mean_iou_chain(p, t, per_class=bool(opt), **kw)
            score += s.mean(0) if opt else s.mean()
        else:
            score += osg.generalized_dice_chain(p, t, weight_type=sc.WEIGHTS[opt % 3], per_class=opt >= 3, **kw).sum(dim=0)
    if kind == 0:
        return {"score": score, "num_batches": torch.tensor(len(c["batches"]))}
    return {"score": score, "samples": torch.zeros(1) + sum(p.shape[0] for p, _ in c["batches"])}


def test_golden_covers_what_it_should(golden):
    metas = np.stack([golden[f"case{k}/meta"] for k in range(int(golden["n_cases"]))])
    kind, index, c, bg, opt, nb, code, layout = metas.T
    assert set(kind) == {0, 1, 2} and set(index) == {0, 1} and set(bg) == {0, 1} and set(layout) == {0, 1}
    assert set(code) >= {0, 1, 2, 3, 4}
    assert set(opt[kind == 1]) == set(range(5)) and set(opt[kind == 2]) == set(range(6)) and set(opt[kind == 0]) == {0, 1}
    assert (nb > 1).any()
    ndims = {golden[f"case{k}/preds0"].ndim - (1 - int(metas[k, 1])) for k in range(len(metas))}
    assert ndims >= {2, 3, 4}  # [N, d], [N, H, W], [N, D, H, W] after the class axis
    u8 = [k for k in range(len(metas)) if metas[k, 6] == 2 and golden[f"case{k}/preds0"].max() > 1]
    assert u8, "non-binary uint8 case missing"


def test_chain_reproduces_the_reference_states(golden):
    for key, c in sc.cases(golden):
        got = _chain_states(c, golden, key)
        for name, value in got.items():
            want = golden[f"{key}/{name}"]
            assert np.array_equal(sc.as_np(value).reshape(want.shape), want), (key, name)


def test_numpy_counts_equal_the_chain_counts(golden):
    for key, c in sc.cases(golden):
        for p, t in c["batches"]:
            pn, tn = p.numpy(), t.numpy()
            for product in ("and", "mul"):
                if product == "and" and p.is_floating_point():
                    continue
                want = osg.counts_chain(p, t, c["num_classes"], c["include_background"], c["index"], product)
                got = osg.counts(pn, tn, c["num_classes"], c["include_background"], c["index"], product)
                for w, g in zip(want, got):
                    if w.is_floating_point():
                        assert np.array_equal(g.astype(np.float32), w.float().numpy()), key  # exact for these sizes
                    else:
                        assert np.array_equal(g, w.numpy()), (key, product)


def test_float64_epilogues_match_the_reference(golden):
    for key, c in sc.cases(golden):
        p, t = c["batches"][0]
        inter, psum, tsum = osg.counts(p.numpy(), t.numpy(), c["num_classes"], c["include_background"], c["index"],
                                       "and" if c["kind"] == 0 else "mul")
        if c["kind"] == 0:
            got = osg.mean_iou_scores(inter, psum, tsum, bool(c["option"]))
        elif c["kind"] == 1:
            got = osg.dice_scores(2 * inter, psum + tsum, tsum, sc.AVERAGES[c["option"]])
        else:
            got = osg.generalized_dice_scores(inter, psum, tsum, sc.WEIGHTS[c["option"] % 3], c["option"] >= 3)
        want = golden[f"{key}/functional"]
        rtol = 2e-3 if c["dtype"] == torch.float16 else 1e-6
        np.testing.assert_allclose(got, want, rtol=rtol, atol=1e-6, err_msg=key)


def test_index_counts_leave_out_of_range_labels_out():
    p = np.array([[0, 1, 2, -1, 7, 2]])
    t = np.array([[0, 5, 2, 2, -3, 2]])
    inter, psum, tsum = osg.counts(p, t, 3, True, True)
    assert inter.tolist() == [[1, 0, 2]] and psum.tolist() == [[1, 1, 2]] and tsum.tolist() == [[1, 0, 3]]
    inter, _, _ = osg.counts(p, t, 3, False, True)
    assert inter.tolist() == [[0, 2]]
