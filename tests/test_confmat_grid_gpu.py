"""GPU: the vec path of K1 / K1b (csrc/confmat.cu) on both sides of every choice of `vec_grid` against the reference's op
chain run on the same GPU (oracle/multiclass_counts.py), bit for bit.

`vec_grid` gives rows of at least 1 KiB one warp each (a grid of ceil(n / 8) CTAs that the hardware block scheduler hands
out) and keeps one resident wave of a grid-stride loop for shorter rows and for sinks with a per-CTA tail (shared-memory
bins, stat-score totals).  The Python side does not see the grid, so these tests do not assert which grid a launch got: they
run every vec-path sink at the shapes where the choice changes and check the counts.  C = 1000, 512, 504 and 256 put the
row size on both sides of 1 KiB (504 bf16: 1008 B, 512 bf16 and 256 f32: 1024 B, 256 bf16: 512 B).  The row
counts straddle one wave for 5 and for 6 resident CTAs per SM (the occupancy of every vec-path instantiation at 35 to 44
registers); the sinks are the confusion matrix, stat scores (macro: global, shared-memory or deferred fold; micro),
samplewise and argmax.
"""
import pytest
import torch

from oracle import multiclass_counts as om
from tests.test_multiclass_counts_paths_gpu import (DEV, FLOATS, check_argmax, check_confmat, check_samplewise,
                                                    check_stats, path_of, rows, stats_state, targets)
from metrics_b200 import _native

pytestmark = pytest.mark.gpu

WARPS_PER_CTA = 8


def row_counts():
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    counts = {1, 7, 8, 9, 65536, 65536 + 13}
    for per_sm in (5, 6):
        edge = sms * per_sm * WARPS_PER_CTA
        counts |= {edge - 1, edge, edge + 1}
    return sorted(counts)


@pytest.fixture(scope="module")
def batches():
    cache = {}

    def get(C, dtype):
        if (C, dtype) not in cache:
            cache.clear()
            n = 65536 + 13
            cache[(C, dtype)] = rows(n, C, dtype, seed=71), targets(n, C, torch.int64, -1, seed=72)
        return cache[(C, dtype)]

    return get


@pytest.mark.parametrize("dtype", FLOATS, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("C", [1000, 512, 504, 256])
def test_every_vec_sink_on_both_sides_of_the_grid_boundary(C, dtype, batches):
    xs, ts = batches(C, dtype)
    for n in row_counts():
        x, t = xs[:n], ts[:n]
        check_confmat(x, t, C, -1, ("vec", "confmat_global"))
        check_stats(x, t, C, -1, False, path_of("stats", x, t, C))
        check_stats(x, t, C, -1, True, path_of("stats", x, t, C, True))
        assert check_argmax(x) == ("vec_plain", "argmax")
        if n * C <= 1 << 25:
            assert check_samplewise(x, t.clamp(min=0), C, None) == ("vec_plain", "samplewise")


@pytest.mark.parametrize("dtype", FLOATS, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("C", [1000, 256])
def test_eight_resident_batches_back_to_back(C, dtype):
    """Eight distinct batches of 65 549 rows, each sink updated back to back with no host synchronisation in between;
    samplewise on the first 16 384 rows of each (its `[3, N, C]` int64 counts)."""
    n, n_sw = 65536 + 13, 16384
    xs = [rows(n, C, dtype, seed=80 + i) for i in range(8)]
    ts = [targets(n, C, torch.int64, -1, seed=90 + i) for i in range(8)]
    assert path_of("confmat", xs[0], ts[0], C) == ("vec", "confmat_global")
    cm = torch.zeros(C, C, dtype=torch.int64, device=DEV)
    states, ws = stats_state(C, False)
    micro, ws_micro = stats_state(C, True)
    am, sw = [], []
    for x, t in zip(xs, ts):
        _native.multiclass_confmat_update_(cm, x, t, C, -1)
        _native.multiclass_stat_scores_update_(*states, ws, x, t, C, -1, False)
        _native.multiclass_stat_scores_update_(*micro, ws_micro, x, t, C, -1, True)
        am.append(_native.argmax_rows(x))
        sw.append(torch.stack(_native.multiclass_stat_scores_samplewise(x[:n_sw], t[:n_sw], C, -1)))
    want_cm = sum(om.confusion_matrix(x, t, C, -1) for x, t in zip(xs, ts))
    want_st = sum(om.stat_scores(x, t, C, 1, "none", "global", -1) for x, t in zip(xs, ts))
    want_mi = sum(om.stat_scores(x, t, C, 1, "micro", "global", -1) for x, t in zip(xs, ts))
    assert torch.equal(cm, want_cm), int((cm - want_cm).abs().sum())
    assert torch.equal(torch.stack(states), want_st.reshape(4, -1))
    assert torch.equal(torch.stack(micro), want_mi.reshape(4, -1))
    assert not bool(ws.any()) and not bool(ws_micro.any())
    for x, t, got_am, got_sw in zip(xs, ts, am, sw):
        assert torch.equal(got_am, x.argmax(1))
        want_sw = om.stat_scores(x[:n_sw], t[:n_sw], C, 1, "none", "samplewise", -1)
        assert torch.equal(got_sw, want_sw), (got_sw - want_sw).abs().sum((-1, -2)).tolist()


def test_more_than_2_31_scores_on_many_waves():
    """`[2^21 + 3, 1024]` bfloat16 (about 4.3 GB, 262 145 CTAs): confusion matrix and argmax with row offsets past 2^31
    elements; the chain runs in row chunks."""
    n, C = (1 << 21) + 3, 1024
    need = n * C * 2 + (2 << 30)
    if torch.cuda.mem_get_info(DEV)[0] < need:
        pytest.skip(f"needs {need >> 30} GiB of free device memory")
    g = torch.Generator(device=DEV).manual_seed(73)
    x = torch.randn(n, C, generator=g, device=DEV, dtype=torch.bfloat16)
    x[-4096:] = rows(4096, C, torch.bfloat16, seed=74)
    t = torch.randint(-1, C, (n,), generator=g, device=DEV)
    assert x.numel() > 2**31
    assert path_of("confmat", x, t, C) == ("vec", "confmat_global")
    cm = torch.zeros(C, C, dtype=torch.int64, device=DEV)
    _native.multiclass_confmat_update_(cm, x, t, C, -1)
    got = _native.argmax_rows(x)
    want_cm = torch.zeros_like(cm)
    step = 1 << 18
    for r in range(0, n, step):
        want_cm += om.confusion_matrix(x[r: r + step], t[r: r + step], C, -1)
        assert torch.equal(got[r: r + step], x[r: r + step].argmax(1)), r
    assert torch.equal(cm, want_cm), int((cm - want_cm).abs().sum())
