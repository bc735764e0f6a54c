"""The k-way merge's position arithmetic without a GPU: frizbee_b200/csrc/merge_plan.cuh built for the CPU from
tests/harness/merge_plan_harness.cpp.  Through the header's own functions, every run is placed into the slices of the
merged list as k_place does, and the slice exchange's ranges are computed and its received pieces scattered as the merge's
scatter kernel does; both must give the host k-way merge (parallel.merge_runs_host), and the table rows must equal the
host specification's pos0 (parallel.block_bases).  The 2-GPU tests are the only GPU runs of these forms, so this is their
check on a machine with fewer GPUs."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from frizbee_b200 import MATCH_DTYPE, parallel
from frizbee_b200.types import SortStrategy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "harness", "merge_plan_harness.cpp")
LIB = os.path.join(ROOT, "tests", "harness", "libmerge_plan_harness.so")
DEPS = [SRC, os.path.join(ROOT, "frizbee_b200", "csrc", "merge_plan.cuh")]
NO_LIMIT = 2**64 - 1


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", LIB, SRC], check=True)
    L = C.CDLL(LIB)
    vp, u64 = C.c_void_p, C.c_uint64
    L.h_tables.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp]
    L.h_tables.restype = None
    L.h_place.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, u64, vp]
    L.h_exchange.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, u64, vp, vp]
    return L


def scores(kind, n, nb, rng):
    """Scores whose order the bins keep: below the last bin, or past it all tied (a clamped top bin)."""
    if kind == "tied":
        return np.full(n, 7, dtype=np.uint16)
    s = rng.integers(0, max(nb - 1, 1), n)
    if kind == "clamped":
        s[rng.random(n) < 0.2] = nb - 1 + 37
    return s.astype(np.uint16)


def make_runs(full, world, sort, skew, rng):
    runs = []
    for lo, hi in parallel.shard_bounds(len(full), world):
        r = full[lo:hi]
        if skew and lo < hi and rng.random() < 0.3:   # a skewed shard: drop most of its matches
            r = r[rng.random(len(r)) < 0.1]
        if sort.is_reversed():
            r = r[::-1]
        if sort.is_by_score():
            r = r[np.argsort(-r["score"].astype(np.int64), kind="stable")]
        runs.append(np.ascontiguousarray(r))
    return runs


def host_gt(runs, nb):
    gt = np.zeros((len(runs), nb), dtype=np.int64)
    for q, r in enumerate(runs):
        hist = np.bincount(np.minimum(r["score"].astype(np.int64), nb - 1), minlength=nb)
        gt[q] = hist[::-1].cumsum()[::-1] - hist
    return gt


def cases(world, sort, rng):
    """(runs, bins) for empty, skewed, all-tied and random runs, runs shorter than the world, and 1 / 512 / 1024 bins
    (the device uses a one-bin table for the index-ordered sorts, and a one-bin table keeps a score order only when tied)."""
    for nb in ((1, 512, 1024) if sort.is_by_score() else (1,)):
        kinds = ("tied",) if nb == 1 and sort.is_by_score() else ("random", "clamped", "tied")
        for kind in kinds:
            for n, skew in ((0, False), (world - 1, False), (1000, False), (1000, True), (37, True)):
                full = np.zeros(n, dtype=MATCH_DTYPE)
                full["index"] = np.arange(n)
                full["score"] = scores(kind, n, nb, rng)
                full["exact"] = rng.integers(0, 2, n)
                yield make_runs(full, world, sort, skew, rng), nb, kind


def limits(merged, nb):
    """None, 0, 1, K' > total, and K' cut inside a tied block (two equal scores on either side of the cut)."""
    out = [None, 0, 1, len(merged) + 5]
    b = np.minimum(merged["score"].astype(np.int64), nb - 1)
    tied = np.nonzero(b[1:] == b[:-1])[0]
    if len(tied):
        out.append(int(tied[len(tied) // 2]) + 1)
    return out


@pytest.mark.parametrize("world", [1, 2, 3, 8, 64])
@pytest.mark.parametrize("sort", list(SortStrategy))
def test_merge_plan_equals_the_k_way_merge(H, world, sort):
    rng = np.random.default_rng(1000 * world + int(sort))
    rev = int(sort.is_reversed())
    checked = 0
    for runs, nb, kind in cases(world, sort, rng):
        counts = np.array([len(r) for r in runs], dtype=np.uint64)
        cat = np.ascontiguousarray(np.concatenate(runs)) if len(runs) else np.zeros(0, dtype=MATCH_DTYPE)
        merged = parallel.merge_runs_host(runs, sort)
        # the table rows: pos0 of the host specification, gt of the runs
        rows = np.zeros((world, 2, nb), dtype=np.uint32)
        H.h_tables(cat.ctypes.data, counts.ctypes.data, world, nb, rev, rows.ctypes.data)
        gt = host_gt(runs, nb)
        assert np.array_equal(rows[:, 0], parallel.block_bases(gt, counts, bool(rev))), (world, sort, nb, kind)
        assert np.array_equal(rows[:, 1], gt)
        for limit in limits(merged, nb):
            kp = len(merged) if limit is None else min(limit, len(merged))
            want = merged[:kp]
            lim = NO_LIMIT if limit is None else limit
            placed = np.zeros(kp, dtype=MATCH_DTYPE)
            assert H.h_place(cat.ctypes.data, counts.ctypes.data, world, nb, rev, lim, placed.ctypes.data) == 0, (world, sort, nb, kind, limit)
            assert np.array_equal(placed, want), (world, sort, nb, kind, limit)
            sliced = np.zeros(kp, dtype=MATCH_DTYPE)
            A = np.zeros((world, world + 1), dtype=np.uint64)
            assert H.h_exchange(cat.ctypes.data, counts.ctypes.data, world, nb, rev, lim, sliced.ctypes.data, A.ctypes.data) == 0, \
                (world, sort, nb, kind, limit)
            assert np.array_equal(sliced, want), (world, sort, nb, kind, limit)
            # a run's pieces tile its kept prefix in slice order
            assert np.all(np.diff(A.astype(np.int64), axis=1) >= 0) and np.all(A[:, 0] == 0)
            assert int(A[:, world].sum()) == kp
            checked += 1
    assert checked > 0
