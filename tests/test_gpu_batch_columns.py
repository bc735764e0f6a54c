"""The batched column call on the GPU (frz_match_list_batch_columns): for every query j, its rows, n_out, n_total and group
counts must be exactly what its own frz_match_list_columns call returns.  Covered: 1-4 columns, empty matchers in some
columns, batched-class queries mixed with fallback ones (negated, multi-pattern, literal, unicode and long-needle column
matchers), every strategy, k from 0 past 1024, per-query and shared subsets, boosts and groups made on any column,
per_group 1, 3, 32 and no cap, rows removed in later columns, appends, survivor lists that overflow, sub-batch boundaries,
repeated matchers and columns, and the device memory the call holds.  Needs a CUDA device."""
import ctypes as C
import random

import numpy as np
import pytest

import frizbee_b200 as F
from collapsing import GROUP_NONE
from frizbee_b200.types import CaseMatching, Config, Matching, Pattern, Scoring, SortStrategy
from scorings import scorings
from test_gpu_batch_scoped import corpus_list, limits, needle_from  # noqa: F401

pytestmark = pytest.mark.gpu

PER_GROUP = [1, 3, 32, None]


def column_matcher(rows, rng, scs, kind, typos=(0, 1, 2, 3, 15, None)):
    """A matcher over one column and its class: "batch" (the batched class), "empty" or "fallback"."""
    cfg = Config(max_typos=rng.choice(typos), casing=rng.choice(list(CaseMatching)),
                 sort=rng.choice(list(SortStrategy)), emulate_lanes=rng.choice([16, 32, 64]), scoring=rng.choice(scs))
    if kind == "empty":
        return F.Matcher("", cfg), "empty"
    if kind == "negated":
        return F.Matcher([Pattern(needle_from(rows, rng, 1, 4)), Pattern("zz", negated=True)], cfg), "fallback"
    if kind == "multi":
        return F.Matcher([Pattern(needle_from(rows, rng, 1, 4)), Pattern(needle_from(rows, rng, 1, 3))], cfg), "fallback"
    if kind == "literal":
        return F.Matcher(needle_from(rows, rng, 1, 4), cfg.with_(matching=rng.choice(
            [Matching.Exact, Matching.Prefix, Matching.Suffix, Matching.Substring]))), "fallback"
    if kind == "unicode":
        return F.Matcher(needle_from(rows, rng, 1, 3) + "é", cfg), "fallback"
    if kind == "long":
        return F.Matcher("f" * rng.randrange(65, 120), cfg.with_(max_typos=None, scoring=Scoring())), "fallback"
    n = rng.choice([1, 2, 3, 5, 8, 12, 20, 40, 64])
    return F.Matcher(needle_from(rows, rng, n, n) if n <= 12 else ("foo_bar" * 10)[:n], cfg), "batch"


FALLBACKS = ["negated", "multi", "literal", "unicode", "long"]


def queries(cols_rows, q, seed, fallbacks=True, empties=True, typos=(0, 1, 2, 3, 15, None)):
    """q queries of one matcher per column; returns the matchers and how many queries are of the batched class (every
    column batched-class or empty, at least one pattern) once F.batch_limits sets a row limit (by default a query with a
    typo budget runs its single call)."""
    rng = random.Random(seed)
    scs = scorings(seed, 8, 64)
    ms, nb = [], 0
    for j in range(q):
        row, classes = [], []
        for rows in cols_rows:
            r = rng.random()
            kind = ("empty" if empties and r < 0.15 else
                    FALLBACKS[j % len(FALLBACKS)] if fallbacks and r > 0.93 else "batch")
            m, cls = column_matcher(rows, rng, scs, kind, typos)
            row.append(m)
            classes.append(cls)
        ms.append(row)
        nb += "fallback" not in classes and "batch" in classes
    return ms, nb


def make_columns(n, n_cols, seed):
    cols_rows = [corpus_list(n, seed=seed + c, long_every=97 if c == 1 else 0) for c in range(n_cols)]
    return cols_rows, [F.Corpus.from_list(r) for r in cols_rows]


def check(ms, cols, k, sort=SortStrategy.ScoreThenIndexAsc, subsets=None, boosts=None, groups=None, per_group=1, batched=None,
          overflowed=0, counts=True):
    """Every query equals its own frz_match_list_columns call; `batched` of them ran the batched kernels."""
    res = F.match_list_batch_columns(ms, cols, k, sort, subsets=subsets, boosts=boosts, groups=groups, per_group=per_group,
                                     counts=counts)
    rows, n_out, n_total = res[:3]
    last = F.batch_last()
    if batched is not None:
        assert last["batched"] == batched and last["overflowed"] == overflowed, (last, batched)
    pgs = per_group if isinstance(per_group, list) else [per_group] * len(ms)
    for j, mj in enumerate(ms):
        s = subsets[j] if subsets else None
        b = boosts[j] if boosts else None
        g = groups[j] if groups else None
        want = F.match_list_columns(mj, cols, k, sort, subset=s, boost=b, groups=g, per_group=pgs[j], counts=g is not None)
        top, total = want[0], want[1]
        assert n_total[j] == total and n_out[j] == len(top), (j, k, sort, n_total[j], total)
        for f in ("index", "score", "exact"):
            assert np.array_equal(rows[j, :len(top)][f], top[f]), (j, k, sort, f)
        assert not rows[j, len(top):].view(np.uint64).any(), (j, k)   # unused rows are not written
        if counts:
            assert (res[3][j] is None) == (g is None), j
            if g is not None:
                assert np.array_equal(res[3][j], want[2]), (j, k)
    return last


def handles(cols, q, seed):
    """Per query a subset, boost and groups handle (or None), each made on a random column, one of each shared by many
    queries and the others their own."""
    rng = np.random.default_rng(seed)
    n = len(cols[0])
    shared_s = cols[-1].subset(np.flatnonzero(rng.random(n) < 0.5).astype(np.uint32))
    shared_b = cols[-1].boost(rng.integers(-300, 301, n).astype(np.int16))
    ids = rng.integers(0, 40, n).astype(np.uint32)
    ids[rng.random(n) < 0.3] = GROUP_NONE
    shared_g = cols[-1].groups(ids, 40)
    subsets, boosts, groups = [], [], []
    for j in range(q):
        c = cols[int(rng.integers(0, len(cols)))]
        kind = int(rng.integers(0, 8))
        s = shared_s if kind == 1 else c.subset(np.flatnonzero(rng.random(n) < rng.choice([0.0, 0.05, 0.6])).astype(np.uint32)) \
            if kind in (2, 3) else None
        b = shared_b if kind in (3, 4) else c.boost(rng.integers(-1000, 1000, int(rng.integers(0, n + 1))).astype(np.int16)) \
            if kind == 5 else None
        g = shared_g if kind in (4, 6) else c.groups(rng.integers(0, max(n // 50, 1), n).astype(np.uint32), max(n // 50, 1)) \
            if kind in (5, 7) else None
        subsets.append(s)
        boosts.append(b)
        groups.append(g)
    return subsets, boosts, groups


@pytest.mark.parametrize("sort", list(SortStrategy), ids=lambda s: s.name)
@pytest.mark.parametrize("n_cols", [1, 2, 3, 4])
def test_mixed_queries_every_strategy(n_cols, sort, limits):
    """Batched-class, empty-column and fallback queries in one call, with and without subsets, boosts and groups."""
    cols_rows, cols = make_columns(3000, n_cols, seed=n_cols)
    ms, nb = queries(cols_rows, 40, seed=n_cols * 10 + int(sort))
    assert nb >= 20
    limits(1 << 18, 2)
    for k in (0, 1, 50):
        check(ms, cols, k, sort, batched=nb)
    subsets, boosts, groups = handles(cols, len(ms), seed=n_cols)
    per_group = [PER_GROUP[j % 4] for j in range(len(ms))]
    check(ms, cols, 50, sort, subsets, boosts, groups, per_group, batched=nb)
    check(ms, cols, 50, sort, subsets, boosts, groups, 3, batched=nb, counts=False)


def test_default_limits_and_k(limits):
    """With the default limits a call batches from 32 batched-class queries on, those whose every pattern has max_typos = 0;
    k = 1024 batches, k = 1025 runs the single calls."""
    cols_rows, cols = make_columns(5000, 2, seed=7)
    ms, nb = queries(cols_rows, 40, seed=7, fallbacks=False, empties=False, typos=(0,))
    assert nb == 40
    typo, _ = queries(cols_rows, 40, seed=8, fallbacks=False, empties=False, typos=(1,))
    check(typo, cols, 10, batched=0)
    check(ms[:31], cols, 10, batched=0)
    check(ms, cols, 10, batched=40)
    check(ms, cols, 1024, SortStrategy.ScoreThenIndexDesc, batched=40)
    check(ms, cols, 1025, batched=0)
    subsets, boosts, groups = handles(cols, len(ms), seed=7)
    check(ms, cols, 1024, SortStrategy.IndexAsc, subsets, boosts, groups, None, batched=40)


def test_every_column_empty_runs_the_single_call(limits):
    cols_rows, cols = make_columns(2000, 2, seed=8)
    limits(1 << 18, 2)
    ms = [[F.Matcher("", Config()), F.Matcher("", Config())] for _ in range(8)]
    check(ms, cols, 10, batched=0)
    cols[1].remove(np.arange(0, 2000, 3, dtype=np.uint32))
    check(ms, cols, 10, SortStrategy.IndexDesc, batched=0)


def test_removed_rows_in_later_columns(limits):
    """Rows removed in column 1 (with patterns) and column 2 (an empty matcher for some queries) leave every query."""
    cols_rows, cols = make_columns(4000, 3, seed=9)
    ms, nb = queries(cols_rows, 48, seed=9, fallbacks=False)
    limits(1 << 18, 2)
    cols[1].remove(np.arange(5, 4000, 7, dtype=np.uint32))
    cols[2].remove(np.arange(0, 4000, 11, dtype=np.uint32))
    for sort in SortStrategy:
        check(ms, cols, 50, sort, batched=nb)
    subsets, boosts, groups = handles(cols, len(ms), seed=9)
    check(ms, cols, 50, SortStrategy.ScoreThenIndexAsc, subsets, boosts, groups, 1, batched=nb)
    # an empty matcher on column 2 for every query: its live rows are folded in
    rng, scs = random.Random(9), scorings(9, 8, 64)
    ms2 = [[column_matcher(cols_rows[0], rng, scs, "batch")[0], column_matcher(cols_rows[1], rng, scs, "batch")[0],
            F.Matcher("", Config())] for _ in range(40)]
    check(ms2, cols, 50, SortStrategy.IndexAsc, batched=40)
    check(ms2, cols, 50, SortStrategy.ScoreThenIndexDesc, batched=40)
    # replaced rows come back
    cols[1].replace_list(np.arange(5, 4000, 14, dtype=np.uint32), ["foo_bar"] * len(range(5, 4000, 14)))
    check(ms, cols, 50, SortStrategy.ScoreThenIndexDesc, batched=nb)


def test_appends(limits):
    """An append that reaches every column keeps every query equal; one that reaches some columns only is refused."""
    cols_rows, cols = make_columns(3000, 2, seed=10)
    ms, nb = queries(cols_rows, 40, seed=10, fallbacks=False)
    limits(1 << 18, 2)
    for c in cols:
        c.append_list(corpus_list(500, seed=99))
    check(ms, cols, 50, batched=nb)
    cols[0].append_list(["foo"] * 10)
    with pytest.raises(F.FrizbeeError):
        F.match_list_batch_columns(ms, cols, 10)
    cols[1].append_list(["bar"] * 10)
    check(ms, cols, 50, batched=nb)


def test_overflowing_survivor_lists_give_equal_results(limits):
    """Every row of column 1 survives a one-byte needle with one typo: the batched lists (max(n / 4, 65536) records per
    class) overflow in a column other than the first, and the sub-batch runs again query by query."""
    n = 200_000
    cols = [F.Corpus.from_list(corpus_list(n, seed=11)), F.Corpus.from_list(["ab"] * n)]
    limits(1 << 18, 2)
    sorts = list(SortStrategy)
    ms = [[F.Matcher("foo"[: 1 + j % 3], Config(max_typos=0, sort=sorts[j % 4])), F.Matcher("ab"[j % 2], Config(max_typos=1))]
          for j in range(8)]
    last = check(ms, cols, 10, batched=0, overflowed=8)
    assert last["sub_batches"] == 1
    # queries that cannot overflow share the sub-batch and run again with it
    ms2 = ms + [[F.Matcher("foo", Config(max_typos=0)), F.Matcher("", Config())] for _ in range(4)]
    check(ms2, cols, 10, batched=0, overflowed=12)


@pytest.mark.parametrize("q", [64, 65, 130])
def test_sub_batch_boundaries(q, limits):
    cols_rows, cols = make_columns(3000, 2, seed=q)
    ms, nb = queries(cols_rows, q, seed=q, fallbacks=False, empties=False)
    assert nb == q
    limits(1 << 18, 2)
    last = check(ms, cols, 20, batched=nb)
    assert last["sub_batches"] == -(-nb // 64)


def test_repeated_matchers_and_columns(limits):
    cols_rows, cols = make_columns(3000, 1, seed=12)
    c = cols[0]
    limits(1 << 18, 2)
    m = F.Matcher("foo", Config(max_typos=1))
    e = F.Matcher("", Config())
    ms = [[m, m, e]] * 6 + [[m, e, m]] * 6
    check(ms, [c, c, c], 30, batched=12)
    check(ms, [c, c, c], 30, SortStrategy.IndexDesc, subsets=[c.subset(np.arange(0, 3000, 2, dtype=np.uint32))] * 12, batched=12)


def _bytes():
    L = F.lib()
    L.frz_debug_device_bytes.restype = C.c_uint64
    L.frz_debug_device_bytes.argtypes = []
    L.frz_debug_device_bytes_peak.restype = C.c_uint64
    L.frz_debug_device_bytes_peak.argtypes = [C.c_int]
    return L


def test_device_memory_returns(limits):
    cols_rows, cols = make_columns(20000, 2, seed=13)
    ms, nb = queries(cols_rows, 64, seed=13, fallbacks=False, empties=False)
    limits(1 << 18, 2)
    F.match_list_batch_columns(ms, cols, 10)   # the corpora's staging and the matchers' first calls
    start = _bytes().frz_debug_device_bytes()
    F.match_list_batch_columns(ms, cols, 10)
    assert F.batch_last()["batched"] == nb
    assert _bytes().frz_debug_device_bytes() == start
