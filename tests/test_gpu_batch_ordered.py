"""The batched call with per-query attributes on the GPU (frz_match_list_batch_ordered): for every query j, its rows, n_out,
n_total and group counts must be exactly what its single-query call returns (frz_match_list_ordered_collapsed with an
attribute and groups, frz_match_list_ordered with an attribute alone, else query j of frz_match_list_batch_collapsed),
across every order and sort strategy, k on both sides of the batched limit, shared and per-query attributes, subsets
(one filled by Corpus.where), boosts and groups, corpora and attributes edited after the handles were made, calls mixing
ordered, unordered and fallback queries, survivor lists that overflow, the launches of an ordered sub-batch, and the
device memory the call holds.  Needs a CUDA device."""
import ctypes as C
import random

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200.types import Config, Order, SortStrategy
from test_gpu_batch_collapsed import PER_GROUP, group_shapes, single as single_collapsed
from test_gpu_batch_scoped import batch_matchers, corpus_list, limits, needle_from, scopes_for  # noqa: F401
from test_gpu_ordered import attr_values

pytestmark = pytest.mark.gpu

ORDERS = list(Order)
SORTS = list(SortStrategy)
KINDS = ["nulls", "ties", "timestamps", "extremes", "short"]


def ordered_matchers(rows, q, seed):
    """q batched-class matchers: query j has sort strategy SORTS[j % 4], needles of 1-12 bytes and typo budgets 0-2 and
    None (every row-count here is below 65536, where max_typos=None batches too)."""
    rng = random.Random(seed)
    out = []
    for j in range(q):
        n = rng.choice([1, 2, 3, 5, 8, 12])
        cfg = Config(max_typos=rng.choice([0, 1, 2, None]), sort=SORTS[j % 4], emulate_lanes=32)
        out.append(F.Matcher(needle_from(rows, rng, n, n), cfg))
    return out


def single(m, corpus, k, a, order, s, b, g, pg):
    """The query's single-query call: (rows, total, counts or None)."""
    if a is None:
        return single_collapsed(m, corpus, k, s, b, g, pg)
    if g is None:
        return (*m.match_list_ordered_array(corpus, a, order, k, subset=s, boost=b), None)
    return m.match_list_ordered_array(corpus, a, order, k, subset=s, boost=b, groups=g, per_group=pg, counts=True)


def check(ms, corpus, k, attrs, orders, subsets=None, boosts=None, groups=None, per_group=1, batched=None, overflowed=0,
          counts=True):
    """Every query equals its single-query call, and `batched` of them were answered by the batched kernels."""
    res = F.match_list_batch_ordered(ms, corpus, k, attrs, orders, subsets=subsets, boosts=boosts, groups=groups,
                                     per_group=per_group, counts=counts)
    rows, n_out, n_total = res[:3]
    last = F.batch_last()
    if batched is not None:
        assert last["batched"] == batched and last["overflowed"] == overflowed, (last, batched)
    q = len(ms)
    at = attrs if isinstance(attrs, list) else [attrs] * q
    od = orders if isinstance(orders, list) else [orders] * q
    pgs = per_group if isinstance(per_group, list) else [per_group] * q
    for j, m in enumerate(ms):
        g = groups[j] if groups else None
        top, total, cnt = single(m, corpus, k, at[j], od[j], subsets[j] if subsets else None, boosts[j] if boosts else None, g, pgs[j])
        assert n_total[j] == total and n_out[j] == len(top), (j, k, n_total[j], total, n_out[j], len(top))
        for f in ("index", "score", "exact"):
            assert np.array_equal(rows[j, :len(top)][f], top[f]), (j, k, f, od[j], m.config.sort)
        assert not rows[j, len(top):].view(np.uint64).any(), (j, k)   # unused rows are not written
        if counts:
            assert (res[3][j] is None) == (g is None), j
            if g is not None:
                assert np.array_equal(res[3][j], cnt), (j, k)
    return last


def per_query_attrs(corpus, q, seed):
    rng = np.random.default_rng(seed)
    return [corpus.attr(attr_values(KINDS[j % len(KINDS)], len(corpus), rng)) for j in range(q)]


def test_orders_strategies_and_k(limits):
    """Every order under every sort strategy, per-query attributes of every shape (nulls, ties, int64 extremes, shorter
    than the corpus), alone and with subsets and boosts; k of 0, 1, 10 and 1024 batched, 1025 on the single-query calls."""
    rows = corpus_list(4000, seed=21)
    corpus = F.Corpus.from_list(rows)
    q = 48
    ms = ordered_matchers(rows, q, 21)
    attrs = per_query_attrs(corpus, q, 21)
    orders = [ORDERS[(j // 4) % 4] for j in range(q)]   # with SORTS[j % 4]: every pair
    subsets, boosts, _, _ = scopes_for(corpus, q, seed=21)
    limits(0, 2)
    for k in (0, 1, 10, 1024):
        check(ms, corpus, k, attrs, orders, batched=q)
        check(ms, corpus, k, attrs, orders, subsets, boosts, batched=q)
    check(ms, corpus, 1025, attrs, orders, subsets, boosts, batched=0)   # k > 1024: every query runs its single-query call


@pytest.mark.parametrize("kind", KINDS)
def test_selections_past_the_block_sort(kind, limits):
    """Queries whose rows outnumber the block sort (one- and two-byte needles over 30 000 rows): their rows go through the
    select's passes, over every order and strategy, with subsets, boosts and groups."""
    rows = corpus_list(30000, seed=33)
    corpus = F.Corpus.from_list(rows)
    q = 32
    rng = random.Random(33)
    ms = [F.Matcher(rng.choice(["f", "o", "fo", "oo", "a"]), Config(max_typos=j % 2, sort=SORTS[j % 4])) for j in range(q)]
    attr = corpus.attr(attr_values(kind, len(rows), np.random.default_rng(33)))
    orders = [ORDERS[(j // 4) % 4] for j in range(q)]
    subsets, boosts, _, _ = scopes_for(corpus, q, seed=33)
    g = corpus.groups(np.arange(len(rows), dtype=np.uint32) % 5000, 5000)
    limits(0, 2)
    assert max(len(m.match_list_into_array(corpus)) for m in ms) > 4096
    for k in (1, 10, 1024):
        check(ms, corpus, k, attr, orders, batched=q)
    check(ms, corpus, 100, attr, orders, subsets, boosts, batched=q)
    check(ms, corpus, 100, attr, orders, subsets, boosts, [g if j % 2 else None for j in range(q)], [PER_GROUP[j % 4] for j in range(q)],
          batched=q)


@pytest.mark.parametrize("per_group", PER_GROUP)
def test_groups_and_counts(per_group, limits):
    """Each group shape shared by the queries of a batch, with a shared attribute, subsets and boosts and every order."""
    rows = corpus_list(3000, seed=22)
    corpus = F.Corpus.from_list(rows)
    q = 40
    ms = ordered_matchers(rows, q, 22)
    attr = corpus.attr(attr_values("ties", len(rows), np.random.default_rng(22)))
    orders = [ORDERS[j % 4] for j in range(q)]
    subsets, boosts, _, _ = scopes_for(corpus, q, seed=22)
    limits(0, 2)
    for name, ids, n_groups in group_shapes(len(rows), 22):
        g = corpus.groups(ids, n_groups)
        check(ms, corpus, 10, attr, orders, groups=[g] * q, per_group=per_group, batched=q)
        check(ms, corpus, 300, attr, orders, subsets, boosts, [g] * q, per_group, batched=q)
        g.close()


def test_per_query_groups_and_where_subset(limits):
    """Per-query attributes, groups and caps, and a subset filled from an attribute by Corpus.where."""
    rows = corpus_list(5000, seed=23)
    corpus = F.Corpus.from_list(rows)
    q = 36
    ms = ordered_matchers(rows, q, 23)
    rng = np.random.default_rng(23)
    status = corpus.attr(attr_values("ties", len(rows), rng))
    stamp = corpus.attr(attr_values("timestamps", len(rows), rng))
    sub = corpus.where(status.isin([0, 127]))
    shapes = group_shapes(len(rows), 23)
    groups = [corpus.groups(*shapes[j % len(shapes)][1:]) for j in range(q)]
    per_group = [PER_GROUP[j % 4] for j in range(q)]
    attrs = [stamp if j % 2 else status for j in range(q)]
    limits(0, 2)
    check(ms, corpus, 10, attrs, Order.AttrDesc, [sub] * q, None, groups, per_group, batched=q)
    check(ms, corpus, 50, attrs, [ORDERS[j % 4] for j in range(q)], [sub if j % 3 else None for j in range(q)], None, groups,
          per_group, batched=q)


@pytest.mark.parametrize("forced", [False, True], ids=["default-limits", "batched-from-2"])
def test_mixed_calls(forced, limits):
    """Ordered, unordered and fallback queries (multi-pattern, negated, literal, unicode, long and empty needles) in one
    call, with and without groups: the ordered and unordered batched queries run in sub-batches of their own."""
    rows = corpus_list(5000, seed=24, long_every=97)
    corpus = F.Corpus.from_list(rows)
    q = 70
    ms, nb = batch_matchers(rows, q, seed=24)
    rng = np.random.default_rng(24)
    attr = corpus.attr(attr_values("timestamps", len(rows), rng))
    attrs = [attr if j % 2 else None for j in range(q)]
    subsets, boosts, _, _ = scopes_for(corpus, q, seed=25)
    shapes = group_shapes(len(rows), 24)
    groups = [None if j % 3 == 0 else corpus.groups(*shapes[j % len(shapes)][1:]) for j in range(q)]
    per_group = [PER_GROUP[j % 4] for j in range(q)]
    if forced:
        limits(0, 2)
    want = nb if nb >= (2 if forced else 32) else 0
    for k in (0, 10):
        last = check(ms, corpus, k, attrs, [ORDERS[j % 4] for j in range(q)], subsets, boosts, groups, per_group, want)
        if want:
            assert last["sub_batches"] >= 2, last   # one ordered, one unordered at the least


def test_corpus_and_attribute_edits(limits):
    """The same handles after removed, replaced and appended rows, and after Attr.set gives rows new values."""
    n = 5 * 1024 + 300
    rows = corpus_list(n, seed=26, long_every=53)
    corpus = F.Corpus.from_list(rows)
    q = 40
    ms = ordered_matchers(rows, q, 26)
    attrs = per_query_attrs(corpus, q, 26)
    subsets, boosts, _, _ = scopes_for(corpus, q, seed=26)
    shapes = group_shapes(n, 26)
    groups = [None if j % 4 == 3 else corpus.groups(*shapes[j % len(shapes)][1:]) for j in range(q)]
    per_group = [PER_GROUP[j % 4] for j in range(q)]
    orders = [ORDERS[j % 4] for j in range(q)]
    limits(0, 2)
    args = (attrs, orders, subsets, boosts, groups, per_group)
    check(ms, corpus, 10, *args, batched=q)
    corpus.remove(np.arange(0, n, 3, dtype=np.uint32))
    check(ms, corpus, 10, *args, batched=q)
    corpus.replace_list(np.arange(1, n, 7, dtype=np.uint32), ["foo_bar"] * len(range(1, n, 7)))
    check(ms, corpus, 10, *args, batched=q)
    corpus.append_list(corpus_list(1500, seed=27))
    check(ms, corpus, 10, *args, batched=q)
    rng = np.random.default_rng(27)
    new = np.arange(n, n + 1500, dtype=np.uint32)
    for a in attrs[:6]:
        which = np.concatenate([new, rng.choice(n, 200, replace=False).astype(np.uint32)])
        a.set(which, rng.integers(-50, 50, len(which)).astype(np.int64))
    check(ms, corpus, 10, *args, batched=q)


def test_no_attributes_equals_match_list_batch_collapsed(limits):
    """attrs None (or a list of None) is match_list_batch_collapsed, with the same launches."""
    rows = corpus_list(4000, seed=28)
    corpus = F.Corpus.from_list(rows)
    ms, nb = batch_matchers(rows, 70, seed=28, with_fallbacks=False)
    subsets, boosts, _, _ = scopes_for(corpus, len(ms), seed=28)
    g = corpus.groups(np.arange(len(rows), dtype=np.uint32) % 40, 40)
    groups = [g if j % 2 else None for j in range(len(ms))]
    limits(0, 2)
    want = F.match_list_batch_collapsed(ms, corpus, 10, groups, 3, subsets=subsets, boosts=boosts, counts=True)
    last = F.batch_last()
    assert last["batched"] == nb
    for attrs in (None, [None] * len(ms)):
        got = F.match_list_batch_ordered(ms, corpus, 10, attrs, subsets=subsets, boosts=boosts, groups=groups, per_group=3, counts=True)
        assert F.batch_last() == last
        for x, y in zip(want[:3], got[:3]):
            assert np.array_equal(x, y)
        assert all((a is None and b is None) or np.array_equal(a, b) for a, b in zip(want[3], got[3]))


def test_launches_do_not_depend_on_q(limits):
    """An ordered sub-batch of 2 queries and one of 40 (one matcher configuration: the same kernel variants) make the same
    launches, grouped or not."""
    rows = corpus_list(3000, seed=29)
    corpus = F.Corpus.from_list(rows)
    attr = corpus.attr(attr_values("timestamps", len(rows), np.random.default_rng(29)))
    g = corpus.groups(np.arange(len(rows), dtype=np.uint32) % 100, 100)
    limits(0, 2)
    for groups in (None, g):
        seen = set()
        for q in (2, 40):
            ms = [F.Matcher("foo", Config(max_typos=1)) for _ in range(q)]
            last = check(ms, corpus, 10, attr, Order.AttrDesc, groups=[groups] * q if groups else None, per_group=2, batched=q)
            assert last["sub_batches"] == 1, last
            seen.add(last["launches"])
        assert len(seen) == 1, seen


def test_overflowing_survivor_lists_give_equal_results():
    """Every row survives a one-byte needle with one typo: the per-query lists of the batched path overflow, and the
    sub-batch runs again query by query through the ordered single-query calls."""
    n = 200_000
    corpus = F.Corpus.from_list(["ab"] * n)
    ms = [F.Matcher(c, Config(max_typos=1, sort=s)) for c, s in zip("ab" * 20, SORTS * 10)]
    rng = np.random.default_rng(30)
    attr = corpus.attr(attr_values("timestamps", n, rng))
    subsets, boosts, _, _ = scopes_for(corpus, len(ms), seed=30)
    g = corpus.groups(rng.integers(0, 1000, n).astype(np.uint32), 1000)
    check(ms, corpus, 10, attr, [ORDERS[j % 4] for j in range(len(ms))], subsets, boosts, [g if j % 2 else None for j in range(len(ms))],
          [PER_GROUP[j % 4] for j in range(len(ms))], batched=0, overflowed=len(ms))


def test_handles_of_another_corpus_are_refused():
    rows = corpus_list(500, seed=31)
    a, b = F.Corpus.from_list(rows), F.Corpus.from_list(rows)
    ms = ordered_matchers(rows, 4, 31)
    aa, ab = a.attr(np.arange(len(rows))), b.attr(np.arange(len(rows)))
    with pytest.raises(F.FrizbeeError) as e:
        F.match_list_batch_ordered(ms, a, 10, [aa, ab, None, None])
    assert e.value.status == 1
    with pytest.raises(F.FrizbeeError) as e:
        F.match_list_batch_ordered(ms, a, 10, aa, [0, 1, 2, 4])
    assert e.value.status == 1
    check(ms, a, 10, aa, Order.ScoreThenAttrAsc, batched=0)


def _bytes():
    L = F.lib()
    L.frz_debug_device_bytes.restype = C.c_uint64
    L.frz_debug_device_bytes.argtypes = []
    return L


def test_device_memory_returns(limits):
    rows = corpus_list(20000, seed=32)
    corpus = F.Corpus.from_list(rows)
    q = 200
    ms = ordered_matchers(rows, q, 32)
    attrs = per_query_attrs(corpus, q, 32)
    shapes = group_shapes(len(rows), 32)
    groups = [None if j % 4 == 3 else corpus.groups(*shapes[j % len(shapes)][1:]) for j in range(q)]
    per_group = [PER_GROUP[j % 4] for j in range(q)]
    orders = [ORDERS[j % 4] for j in range(q)]
    F.match_list_batch_ordered(ms, corpus, 10, attrs, orders, groups=groups, per_group=per_group)   # the corpus's staging first
    start = _bytes().frz_debug_device_bytes()
    F.match_list_batch_ordered(ms, corpus, 10, attrs, orders, groups=groups, per_group=per_group, counts=True)
    assert F.batch_last()["batched"] == q
    assert _bytes().frz_debug_device_bytes() == start
