"""Top-K match_list without a GPU: the host specification of the limited multi-GPU placement (parallel.placement_host with
`limit`) against the truncated k-way merge, and the new entry points' argument checks and missing-device status."""
import ctypes

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200 import parallel
from frizbee_b200.types import Config, SortStrategy


def _run(rng, n, lo_score, hi_score, start):
    """One shard's run, ordered like the GPU leaves it: index order, then a stable score sort for the by-score strategies."""
    r = np.zeros(n, dtype=F.MATCH_DTYPE)
    r["index"] = start + np.sort(rng.choice(10 * max(n, 1), size=n, replace=False)).astype(np.uint32)
    r["score"] = rng.integers(lo_score, hi_score + 1, size=n).astype(np.uint16)
    r["exact"] = rng.integers(0, 2, size=n).astype(np.uint8)
    return r


def _ordered(run, sort):
    if sort.is_reversed():
        run = run[::-1]
    if sort.is_by_score():
        run = run[np.argsort(-run["score"].astype(np.int64), kind="stable")]
    return np.ascontiguousarray(run)


def _runs(seed, sizes, lo_score=0, hi_score=40):
    rng = np.random.default_rng(seed)
    out, start = [], 0
    for n in sizes:
        out.append(_run(rng, n, lo_score, hi_score, start))
        start += 10 * max(n, 1) + 1
    return out


def _check(runs, sort, k):
    ordered = [_ordered(r, sort) for r in runs]
    want = parallel.merge_runs_host(ordered, sort)[:k]
    slices = parallel.placement_host(ordered, sort, limit=k)
    assert len(slices) == len(runs)
    keep = min(k, sum(len(r) for r in runs))
    assert [len(s) for s in slices] == [keep * (p + 1) // len(runs) - keep * p // len(runs) for p in range(len(runs))]
    got = np.concatenate(slices) if slices else np.zeros(0, dtype=F.MATCH_DTYPE)
    assert len(got) == len(want) and np.array_equal(got, want), (sort, k, [len(r) for r in runs])


@pytest.mark.parametrize("sort", list(SortStrategy))
@pytest.mark.parametrize("world", range(1, 9))
def test_placement_limit_equals_truncated_merge(sort, world):
    """Every strategy, world sizes 1-8, K at 0, 1, total - 1, total, total + 5 and a few in between."""
    runs = _runs(world, [300 + 37 * q for q in range(world)])
    total = sum(len(r) for r in runs)
    for k in (0, 1, 2, 17, total // 3, total - 1, total, total + 5):
        _check(runs, sort, k)


@pytest.mark.parametrize("sort", list(SortStrategy))
def test_placement_limit_skewed_and_empty_runs(sort):
    """One run holds almost everything, some runs are empty, and the last run is the only non-empty one."""
    for sizes in ([2000, 0, 3, 0], [0, 0, 0, 500], [0, 0], [1, 0, 0, 0, 0, 0, 0, 0], [0, 900, 0, 7, 0, 0, 1]):
        runs = _runs(len(sizes) + 100, sizes)
        total = sum(sizes)
        for k in sorted({0, 1, max(total - 1, 0), total, total + 5, 2 * total // 3}):
            _check(runs, sort, k)


@pytest.mark.parametrize("sort", [SortStrategy.ScoreThenIndexAsc, SortStrategy.ScoreThenIndexDesc])
def test_placement_limit_inside_a_block_of_tied_scores(sort):
    """Hundreds of matches in every run share the score at position K: the merge order (runs in index order, or reversed)
    decides which of them are kept."""
    rng = np.random.default_rng(5)
    runs, start = [], 0
    for q in range(4):
        r = _run(rng, 400, 0, 0, start)
        r["score"][:150] = 30            # the tied block
        r["score"][150:160] = 50         # a few above it
        r["score"][160:] = rng.integers(0, 20, size=240).astype(np.uint16)
        runs.append(r)
        start += 10 * 400 + 1
    for k in (40, 41, 100, 333, 639, 640, 641):   # 40 score 50, then 600 score 30
        _check(runs, sort, k)


def test_top_entry_points_argument_errors_and_no_device():
    """k > 0 with a null `out` is an argument error; null handles are argument errors; without a device the call reports
    FRZ_ERR_NO_DEVICE — there is no CPU fallback."""
    import torch
    L = parallel.plib()
    n, total = ctypes.c_uint64(), ctypes.c_uint64()
    assert L.frz_match_list_top(None, None, 10, None, ctypes.byref(n), ctypes.byref(total)) == 1   # FRZ_ERR_INVALID_ARG
    assert L.frz_match_list_parallel_top(None, None, 0, None, 10, None, ctypes.byref(n), None) == 1
    assert L.frz_match_list_parallel_top(None, None, 0, None, 0, None, ctypes.byref(n), None) == 1
    assert L.frz_match_list_parallel_rank_top(None, None, 0, None, 10, None, ctypes.byref(n), None, None) == 1
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    m = F.Matcher("foo", Config())
    with pytest.raises(F.FrizbeeError) as e:
        m.match_list_top_array(["foo", "bar"], 1)
    assert e.value.status_name == "FRZ_ERR_NO_DEVICE" and "no CPU fallback" in str(e.value)
    with pytest.raises(F.FrizbeeError) as e:
        parallel.Comm.local(1)
    assert e.value.status_name == "FRZ_ERR_NO_DEVICE"
    m.close()
