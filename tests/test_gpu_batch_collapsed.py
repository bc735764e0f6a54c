"""The batched call with per-query groups on the GPU (frz_match_list_batch_collapsed): for every query j, its rows, n_out,
n_total and group counts must be exactly what its single-query call returns (frz_match_list_collapsed with groups, else
query j of frz_match_list_batch), across batched-class and fallback queries, group shapes and per-group caps, shared and
per-query handles with subsets and boosts, corpora edited after the handles were made, survivor lists that overflow,
group handles too large for the batched tables, and the device memory the call holds.  Needs a CUDA device."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from collapsing import GROUP_NONE
from frizbee_b200.types import Config, SortStrategy
from test_gpu_batch_scoped import batch_matchers, corpus_list, limits, scopes_for, single as single_scoped  # noqa: F401

pytestmark = pytest.mark.gpu

PER_GROUP = [1, 3, 32, None]


def group_shapes(n, seed):
    """(name, ids, n_groups) group shapes over n rows, those of test_gpu_collapsed.py"""
    rng = np.random.default_rng(seed)
    mixed = rng.integers(0, 40, n).astype(np.uint32)
    mixed[rng.random(n) < 0.3] = GROUP_NONE
    return [("none", np.full(n, GROUP_NONE, np.uint32), 1),
            ("own", np.arange(n, dtype=np.uint32), max(n, 1)),
            ("one", np.zeros(n, np.uint32), 1),
            ("dup", rng.integers(0, max(n // 50, 1), n).astype(np.uint32), max(n // 50, 1)),
            ("short", rng.integers(0, 5, n // 3).astype(np.uint32), 7),    # rows past n // 3 are in no group
            ("mixed", mixed, 40)]


def single(m, corpus, k, s, b, g, pg):
    """The query's single-query call: (rows, total, counts or None)."""
    if g is None:
        return (*single_scoped(m, corpus, k, s, b), None)
    return m.match_list_collapsed_array(corpus, g, k, per_group=pg, subset=s, boost=b, counts=True)


def check(ms, corpus, k, groups, per_group, subsets=None, boosts=None, batched=None, overflowed=0, counts=True):
    """Every query equals its single-query call, and `batched` of them were answered by the batched kernels."""
    res = F.match_list_batch_collapsed(ms, corpus, k, groups, per_group, subsets=subsets, boosts=boosts, counts=counts)
    rows, n_out, n_total = res[:3]
    last = F.batch_last()
    if batched is not None:
        assert last["batched"] == batched and last["overflowed"] == overflowed, (last, batched)
    pgs = per_group if isinstance(per_group, list) else [per_group] * len(ms)
    for j, m in enumerate(ms):
        g = groups[j] if groups else None
        top, total, cnt = single(m, corpus, k, subsets[j] if subsets else None, boosts[j] if boosts else None, g, pgs[j])
        assert n_total[j] == total and n_out[j] == len(top), (j, k, n_total[j], total)
        for f in ("index", "score", "exact"):
            assert np.array_equal(rows[j, :len(top)][f], top[f]), (j, k, f)
        assert not rows[j, len(top):].view(np.uint64).any(), (j, k)   # unused rows are not written
        if counts:
            assert (res[3][j] is None) == (g is None), j
            if g is not None:
                assert np.array_equal(res[3][j], cnt), (j, k)
    return last


def handles_for(corpus, q, seed, shared):
    """Per query a groups handle (or None for every fourth query): one handle shared by all, or one per query."""
    n = len(corpus)
    shapes = group_shapes(n, seed)
    if shared:
        _, ids, n_groups = shapes[5]
        g = corpus.groups(ids, n_groups)
        return [None if j % 4 == 3 else g for j in range(q)]
    return [None if j % 4 == 3 else corpus.groups(*shapes[j % len(shapes)][1:]) for j in range(q)]


@pytest.mark.parametrize("shared", [True, False], ids=["shared", "per-query"])
@pytest.mark.parametrize("forced", [False, True], ids=["default-limits", "batched-from-2"])
@pytest.mark.parametrize("q", [2, 40, 70])
def test_mixed_batches_equal_the_single_query_calls(q, forced, shared, limits):
    """Batched-class and fallback queries (multi-pattern, negated, literal, unicode, long and empty needles) with grouped,
    ungrouped, scoped and ranked queries in one sub-batch, per_group 1, 3, 32 and no cap."""
    rows = corpus_list(5000, seed=q, long_every=97)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, q, seed=q)
    subsets, boosts, _, _ = scopes_for(corpus, q, seed=q + 1)
    groups = handles_for(corpus, q, q, shared)
    per_group = [PER_GROUP[j % 4] for j in range(q)]
    if forced:
        limits(0, 2)
    want = nb if nb >= (2 if forced else 32) else 0
    for k in (0, 1, 10):
        check(ms, corpus, k, groups, per_group, subsets, boosts, want)
    check(ms, corpus, 10, groups, per_group, subsets, boosts, want, counts=False)


@pytest.mark.parametrize("per_group", PER_GROUP)
def test_group_shapes_every_strategy(per_group, limits):
    """Each group shape shared by every query of a batch whose queries cover every sort strategy, typo budget, u8 and
    u16 scores (needles of 1-64 bytes under scorings up to 64), alone and with subsets and boosts."""
    rows = corpus_list(4000, seed=5)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, 48, seed=5, with_fallbacks=False)
    assert nb == len(ms)
    subsets, boosts, _, _ = scopes_for(corpus, len(ms), seed=5)
    limits(0, 2)
    for name, ids, n_groups in group_shapes(len(rows), 5):
        g = corpus.groups(ids, n_groups)
        check(ms, corpus, 10, [g] * len(ms), per_group, batched=nb)
        check(ms, corpus, 300, [g] * len(ms), per_group, subsets, boosts, batched=nb)
        g.close()


def test_some_queries_want_counts(limits):
    """group_counts with NULL entries: only the queries that ask get their counts, the others' arrays stay untouched."""
    rows = corpus_list(3000, seed=6)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, 20, seed=6, with_fallbacks=False)
    shapes = group_shapes(len(rows), 6)
    groups = [corpus.groups(*shapes[j % len(shapes)][1:]) for j in range(len(ms))]
    limits(0, 2)
    q, k = len(ms), 10
    cnt = [np.full(len(g), 7, np.uint32) for g in groups]
    hc = (C.c_void_p * q)(*[c.ctypes.data if j % 3 == 1 else None for j, c in enumerate(cnt)])
    hg = (C.c_void_p * q)(*[g._h.value for g in groups])
    hm = (C.c_void_p * q)(*[m._h.value for m in ms])
    pg = np.array([PER_GROUP[j % 4] or 2**64 - 1 for j in range(q)], np.uint64)
    out = np.zeros((q, k), dtype=F.MATCH_DTYPE)
    n_out, n_total = np.zeros(q, np.uint64), np.zeros(q, np.uint64)
    assert F.lib().frz_match_list_batch_collapsed(hm, q, corpus._h, None, None, hg, pg.ctypes.data, k, out.ctypes.data,
                                                  n_out.ctypes.data, n_total.ctypes.data, hc) == 0
    assert F.batch_last()["batched"] == nb
    for j, m in enumerate(ms):
        top, total, want = single(m, corpus, k, None, None, groups[j], PER_GROUP[j % 4])
        assert n_total[j] == total and np.array_equal(out[j, :n_out[j]], top), j
        assert np.array_equal(cnt[j], want) if j % 3 == 1 else (cnt[j] == 7).all(), j


@pytest.mark.parametrize("n", [0, 700, 5 * 1024 + 300])
def test_corpus_shapes_and_edits(n, limits):
    """The empty corpus, one partial tile, several tiles; then, with the same handles, removed rows, replaced rows, and
    appended rows (in no group until Groups.set gives them one)."""
    rows = corpus_list(n, seed=n, long_every=53)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows or ["foo"], 40, seed=n)
    subsets, boosts, _, _ = scopes_for(corpus, len(ms), seed=n)
    groups = handles_for(corpus, len(ms), n, shared=False)
    per_group = [PER_GROUP[j % 4] for j in range(len(ms))]
    limits(0, 2)
    check(ms, corpus, 10, groups, per_group, subsets, boosts, nb)
    if n:
        corpus.remove(np.arange(0, n, 3, dtype=np.uint32))
        check(ms, corpus, 10, groups, per_group, subsets, boosts, nb)
        corpus.replace_list(np.arange(1, n, 7, dtype=np.uint32), ["foo_bar"] * len(range(1, n, 7)))
        check(ms, corpus, 10, groups, per_group, subsets, boosts, nb)
        corpus.append_list(corpus_list(1500, seed=n + 1))
        check(ms, corpus, 10, groups, per_group, subsets, boosts, nb)
        new = np.arange(n, n + 1500, dtype=np.uint32)
        for g in {id(g): g for g in groups if g is not None}.values():
            g.set(new, (new % len(g)).astype(np.uint32))
        check(ms, corpus, 10, groups, per_group, subsets, boosts, nb)


def test_k_past_the_totals_and_past_the_batched_limit(limits):
    rows = corpus_list(900, seed=8)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, 40, seed=8, with_fallbacks=False)
    groups = handles_for(corpus, len(ms), 8, shared=False)
    limits(0, 2)
    check(ms, corpus, len(rows) + 5, groups, 3, batched=nb)
    check(ms, corpus, 1024, groups, None, batched=nb)
    check(ms, corpus, 1025, groups, 1, batched=0)   # k > 1024: every query runs its single-query call


def test_no_groups_equals_match_list_batch(limits):
    """groups None (or a list of None) equals match_list_batch, with the same launches."""
    rows = corpus_list(4000, seed=12)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, 70, seed=12, with_fallbacks=False)
    subsets, boosts, _, _ = scopes_for(corpus, len(ms), seed=12)
    limits(0, 2)
    want = F.match_list_batch(ms, corpus, 10, subsets=subsets, boosts=boosts)
    last = F.batch_last()
    assert last["batched"] == nb
    for groups in (None, [None] * len(ms)):
        got = F.match_list_batch_collapsed(ms, corpus, 10, groups, subsets=subsets, boosts=boosts, counts=True)
        assert F.batch_last() == last
        for x, y in zip(want, got[:3]):
            assert np.array_equal(x, y)
        assert all(c is None for c in got[3])


def test_overflowing_survivor_lists_give_equal_results():
    """Every row survives a one-byte needle with one typo: the per-query lists of the batched path overflow, and the
    sub-batch runs again query by query through the collapsed single-query calls."""
    n = 200_000
    corpus = F.Corpus.from_list(["ab"] * n)
    ms = [F.Matcher(c, Config(max_typos=1, sort=s)) for c, s in zip("ab" * 20, list(SortStrategy) * 10)]
    subsets, boosts, _, _ = scopes_for(corpus, len(ms), seed=5)
    g = corpus.groups(np.random.default_rng(5).integers(0, 1000, n).astype(np.uint32), 1000)
    check(ms, corpus, 10, [g] * len(ms), [PER_GROUP[j % 4] for j in range(len(ms))], subsets, boosts, batched=0,
          overflowed=len(ms))


def test_groups_past_the_budget_run_the_single_query_call(limits):
    """A handle of 24 M groups does not fit two to a sub-batch: its queries run frz_match_list_collapsed inside the call,
    the rest are batched."""
    rows = corpus_list(3000, seed=13)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, 12, seed=13, with_fallbacks=False)
    big = corpus.groups(np.random.default_rng(13).integers(0, 24_000_000, len(rows)).astype(np.uint32), 24_000_000)
    small = corpus.groups(np.arange(len(rows), dtype=np.uint32) % 50, 50)
    groups = [big if j < 3 else small for j in range(len(ms))]
    limits(0, 2)
    check(ms, corpus, 10, groups, [1, None, 3] + [2] * (len(ms) - 3), batched=nb - 3)


def test_counts_of_many_groups_run_the_single_query_call(limits):
    """A query that wants the counts of more than 2^18 groups runs frz_match_list_collapsed; without counts it is batched."""
    rows = corpus_list(3000, seed=14)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, 12, seed=14, with_fallbacks=False)
    many = corpus.groups(np.random.default_rng(14).integers(0, 300_000, len(rows)).astype(np.uint32), 300_000)
    edge = corpus.groups(np.arange(len(rows), dtype=np.uint32), 1 << 18)
    groups = [many if j < 4 else edge for j in range(len(ms))]
    limits(0, 2)
    check(ms, corpus, 10, groups, 2, batched=nb - 4)
    check(ms, corpus, 10, groups, 2, batched=nb, counts=False)


def test_handles_of_another_corpus_are_refused():
    rows = corpus_list(500, seed=3)
    a, b = F.Corpus.from_list(rows), F.Corpus.from_list(rows)
    ms, _ = batch_matchers(rows, 4, seed=3, with_fallbacks=False)
    ga, gb = a.groups([0, 1, 0]), b.groups([0, 1, 0])
    with pytest.raises(F.FrizbeeError) as e:
        F.match_list_batch_collapsed(ms, a, 10, [ga, gb, None, None])
    assert e.value.status == 1
    check(ms, a, 10, [ga] * 4, 1, batched=0)


def _bytes():
    L = F.lib()
    L.frz_debug_device_bytes.restype = C.c_uint64
    L.frz_debug_device_bytes.argtypes = []
    return L


def test_device_memory_returns(limits):
    rows = corpus_list(20000, seed=9)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, 200, seed=9, with_fallbacks=False)
    groups = handles_for(corpus, len(ms), 9, shared=False)
    per_group = [PER_GROUP[j % 4] for j in range(len(ms))]
    F.match_list_batch_collapsed(ms, corpus, 10, groups, per_group)   # the single-query workspaces first
    start = _bytes().frz_debug_device_bytes()
    F.match_list_batch_collapsed(ms, corpus, 10, groups, per_group, counts=True)
    assert F.batch_last()["batched"] == nb
    assert _bytes().frz_debug_device_bytes() == start
