"""Ordered column calls on the GPU (frz_match_list_columns_ordered).  The contract: the joined rows of the column call
(tests/columns.py's combine: rows live and matching in every column, scores summed with saturation, exact flags ORed) in
index order, ordered by the attribute as tests/ordering.py's order_by_attr orders them (the boost inside the score), then
collapsed by tests/collapsing.py's collapse when groups are given.  Every check compares bit for bit with that
specification over the GPU's own per-column match_list_into: two and three columns, every order and strategy, with and
without groups, a subset or boost made on a later column, columns with removed rows, an empty matcher and an all-negated
column, and the refused calls that need real corpora."""
import numpy as np
import pytest

import frizbee_b200 as F
from collapsing import collapse
from columns import combine
from frizbee_b200.types import Config, Order, SortStrategy
from ordering import order_by_attr
from test_gpu_collapsed import gen, shapes
from test_gpu_ordered import attr_values, expect

pytestmark = pytest.mark.gpu

TILE = 1024
LANES = 32
ORDERS = list(Order)
SORTS = list(SortStrategy)


def cfg(max_typos=0):
    return Config(max_typos=max_typos, emulate_lanes=LANES)


def specification(ms, cols, values, order, sort, members=None, boost_values=None, ids=None, per_group=1, n_groups=None):
    lists = [m.match_list_into_array(c).copy() for m, c in zip(ms, cols)]
    rows = combine(lists, len(cols[0]), members=members)
    L = order_by_attr(rows, values, int(order), sort.is_reversed(), boost_values)
    if ids is None:
        return L, None
    return collapse(L, ids, per_group, n_groups)


def check(ms, cols, attr, values, order, sort, ks=(0, 1, 50, None), subset=None, members=None, boost=None, boost_values=None,
          groups=None, ids=None, per_group=1, ctx=()):
    want, wcounts = specification(ms, cols, values, order, sort, members, boost_values, ids, per_group,
                                  len(groups) if groups is not None else None)
    for k in ks:
        c = ctx + (order, sort.name, per_group, k)
        if groups is None:
            got, total = F.match_list_columns(ms, cols, k, sort, subset=subset, boost=boost, attr=attr, order=order)
        else:
            got, total, counts = F.match_list_columns(ms, cols, k, sort, subset=subset, boost=boost, groups=groups,
                                                      per_group=per_group, counts=True, attr=attr, order=order)
            assert np.array_equal(counts, wcounts), c
        assert total == len(want), (c, total, len(want))
        expect(got, want if k is None else want[:k], c)
    return want


@pytest.fixture(scope="module")
def three():
    cols = [F.Corpus.from_list(gen(3 * TILE + 77, seed)) for seed in (21, 22, 23)]
    yield cols
    for c in cols:
        c.close()


COLUMN_SETS = {
    "two": lambda: [F.Matcher("deadbeef", cfg(1)), F.Matcher("foo", cfg(0))],
    "two-wide": lambda: [F.Matcher("dbf", cfg(None)), F.Matcher("ef", cfg(0))],
    "three": lambda: [F.Matcher("ab", cfg(0)), F.Matcher("dbf", cfg(None)), F.Matcher("e", cfg(0))],
    "empty": lambda: [F.Matcher.from_query("", cfg(0)), F.Matcher("ef", cfg(0))],
    "all-negated": lambda: [F.Matcher("de", cfg(0)), F.Matcher.from_query("!foo !bar", cfg(0))],
}


@pytest.mark.parametrize("name", list(COLUMN_SETS))
def test_orders_strategies_and_groups(three, name):
    ms = COLUMN_SETS[name]()
    cols = three[: len(ms)]
    n = len(cols[0])
    rng = np.random.default_rng(len(name))
    values = attr_values("nulls" if len(ms) == 2 else "ties", n, rng)
    attr = cols[0].attr(values)
    _, ids, n_groups = shapes(n, 11)[5]
    g = cols[-1].groups(ids, n_groups)   # a handle of the last column serves every column
    try:
        want = specification(ms, cols, values, Order.AttrDesc, SortStrategy.IndexAsc)[0]
        assert len(want) > 20, (name, len(want))
        for sort in SORTS:
            for order in ORDERS:
                check(ms, cols, attr, values, order, sort, ctx=(name,))
                for pg in (1, 3, None):
                    check(ms, cols, attr, values, order, sort, (0, 7, None), groups=g, ids=ids, per_group=pg, ctx=(name,))
    finally:
        g.close()
        attr.close()
        for m in ms:
            m.close()


def test_subset_and_boost_of_a_later_column(three):
    ms = COLUMN_SETS["two-wide"]()
    cols = three[:2]
    n = len(cols[0])
    rng = np.random.default_rng(4)
    values = attr_values("timestamps", n, rng)
    attr = cols[1].attr(values)
    members = np.sort(rng.choice(n, n // 2, replace=False)).astype(np.uint32)
    sub = cols[1].subset(members)
    bvals = rng.integers(-200, 201, n).astype(np.int16)
    boost = cols[1].boost(bvals)
    _, ids, n_groups = shapes(n, 12)[3]
    g = cols[1].groups(ids, n_groups)
    try:
        for sort in SORTS:
            for order in ORDERS:
                for s, mem in ((None, None), (sub, members)):
                    for b, bv in ((None, None), (boost, bvals)):
                        check(ms, cols, attr, values, order, sort, (7, None), subset=s, members=mem, boost=b, boost_values=bv,
                              ctx=("plain", s is not None, b is not None))
                        check(ms, cols, attr, values, order, sort, (7, None), subset=s, members=mem, boost=b, boost_values=bv,
                              groups=g, ids=ids, per_group=2, ctx=("grouped", s is not None, b is not None))
    finally:
        for h in (g, boost, sub, attr):
            h.close()
        for m in ms:
            m.close()


def test_columns_with_removed_rows():
    cols = [F.Corpus.from_list(gen(2 * TILE + 50, seed)) for seed in (41, 42, 43)]
    ms = COLUMN_SETS["three"]()
    n = len(cols[0])
    rng = np.random.default_rng(44)
    values = attr_values("extremes", n, rng)
    attr = cols[2].attr(values)
    _, ids, n_groups = shapes(n, 13)[5]
    g = cols[0].groups(ids, n_groups)
    try:
        cols[1].remove(rng.choice(n, 300, replace=False).astype(np.uint32))
        cols[2].remove(rng.choice(n, 200, replace=False).astype(np.uint32))
        for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexDesc):
            for order in ORDERS:
                check(ms, cols, attr, values, order, sort, (5, None))
                check(ms, cols, attr, values, order, sort, (5, None), groups=g, ids=ids, per_group=1)
    finally:
        g.close()
        attr.close()
        for m in ms:
            m.close()
        for c in cols:
            c.close()


def test_refused_calls(three):
    ms = COLUMN_SETS["two"]()
    other = F.Corpus.from_list(gen(100, 5))
    shorter = F.Corpus.from_list(gen(len(three[0]) - 1, 6))
    a_other = other.attr([1])
    attr = three[1].attr([1, 2])
    try:
        with pytest.raises(F.FrizbeeError) as e:   # columns of different lengths
            F.match_list_columns(ms, [three[0], shorter], 5, attr=attr)
        assert e.value.status == 1 and "index space" in str(e.value)
        with pytest.raises(F.FrizbeeError) as e:   # an attribute made on none of the columns
            F.match_list_columns(ms, three[:2], 5, attr=a_other)
        assert e.value.status == 1 and "attribute was made on none" in str(e.value)
        with pytest.raises(F.FrizbeeError) as e:
            F.match_list_columns(ms, three[:2], 5, attr=attr, order=4)
        assert e.value.status == 1
    finally:
        for h in (attr, a_other):
            h.close()
        for c in (other, shorter):
            c.close()
        for m in ms:
            m.close()
