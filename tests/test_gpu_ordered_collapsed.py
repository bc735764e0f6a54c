"""Ordered collapsed calls on the GPU (frz_match_list_ordered_collapsed).  The contract: L is the ordered call's list (the
rows of match_list_into, or of a subset's members, reversed for the *_DESC strategies, sorted stably by tests/ordering.py's
order_by_attr); C keeps, in L's order, the rows in no group and the first per_group rows of each group
(tests/collapsing.py's collapse); the call returns C's first k rows, |C| as the total and L's rows per group as the counts.
Every check compares bit for bit with collapse(order_by_attr(...)) applied to the GPU's own match_list_into (pinned to the
oracle by the parity tests): every order, strategy, per_group and k, subsets (one filled by `where`) and boosts, the
attribute shapes of test_gpu_ordered.py and the group shapes of test_gpu_collapsed.py, the empty matcher ("the latest row
of each group"), every needle class, corpus and handle edits, the survivor-overflow retry, selections on both sides of the
one-block sort, the uncapped call against frz_match_list_ordered, and the device memory the calls hold."""
import numpy as np
import pytest

import frizbee_b200 as F
import test_gpu_survivor_overflow as SO
from collapsing import GROUP_NONE, collapse
from frizbee_b200.types import Config, Order, SortStrategy
from ordering import ATTR_NULL, order_by_attr
from test_gpu_collapsed import shapes
from test_gpu_ordered import attr_values, device_bytes, expect
from test_gpu_ranked import LONG300, gen

pytestmark = pytest.mark.gpu

TILE = 1024
LANES = 32
BLOCK_ROWS = 4096   # kFrzOrderBlockRows
I64_MAX = 2**63 - 1
ORDERS = list(Order)
SORTS = list(SortStrategy)
PER_GROUP = (1, 2, 32, None)
KINDS = ["nulls", "ties", "timestamps", "extremes", "short"]


def cfg(sort, max_typos=0, **kw):
    return Config(max_typos=max_typos, sort=sort, emulate_lanes=LANES, **kw)


def specification(rows, values, order, reversed_, ids, per_group, n_groups, boost_values=None):
    """(C, counts): collapse(order_by_attr(rows, ...)) over the index-ordered rows."""
    return collapse(order_by_attr(rows, values, int(order), reversed_, boost_values), ids, per_group, n_groups)


def check(m, corpus, attr, values, order, groups, ids, per_group, ks, rows, subset=None, boost=None, boost_values=None, ctx=()):
    """The call at every k of ks against the specification over rows (the GPU's own match_list_into, restricted to the
    subset's members when there is one).  "n" in ks is len(rows), "n+5" one past it by 5, "C" the number of kept rows."""
    want, wcounts = specification(rows, values, order, SortStrategy(m.config.sort).is_reversed(), ids, per_group, len(groups),
                                  boost_values)
    for k in ks:
        k = {"n": len(rows), "n+5": len(rows) + 5, "C": len(want)}.get(k, k)
        got, total, counts = m.match_list_ordered_array(corpus, attr, order, k, subset=subset, boost=boost, groups=groups,
                                                        per_group=per_group, counts=True)
        c = ctx + (order, per_group, k)
        assert total == len(want), (c, total, len(want))
        expect(got, want if k is None else want[:k], c)
        assert np.array_equal(counts, wcounts), c
    return want


@pytest.fixture(scope="module")
def small():
    corpus = F.Corpus.from_list(gen(6 * TILE + 321, 11))
    yield corpus
    corpus.close()


@pytest.mark.parametrize("kind", KINDS)
def test_orders_strategies_per_group_and_k(small, kind):
    """Every order × strategy × per_group × k, over every group shape, for one attribute shape."""
    rng = np.random.default_rng(100 + KINDS.index(kind))
    values = attr_values(kind, len(small), rng)
    attr = small.attr(values)
    handles = [(name, ids, small.groups(ids, n_groups)) for name, ids, n_groups in shapes(len(small), 17)]
    try:
        for sort in SORTS:
            m = F.Matcher("deadbeef", cfg(sort, 1))
            into = m.match_list_into_array(small).copy()
            for name, ids, g in handles:
                for order in ORDERS:
                    for pg in PER_GROUP:
                        check(m, small, attr, values, order, g, ids, pg, (0, 1, 7, "n", "n+5", None), into,
                              ctx=(kind, sort.name, name))
            m.close()
    finally:
        for _, _, g in handles:
            g.close()
        attr.close()


def test_subsets_and_boosts(small):
    """A subset, a boost and both (each handle of its own), and a subset filled by `where`, for every order and strategy."""
    rng = np.random.default_rng(3)
    values = attr_values("timestamps", len(small), rng)
    status = attr_values("ties", len(small), rng)
    attr, st = small.attr(values), small.attr(status)
    bvals = rng.integers(-300, 301, len(small)).astype(np.int16)
    boost = small.boost(bvals)
    members = np.sort(rng.choice(len(small), len(small) // 3, replace=False)).astype(np.uint32)
    sub = small.subset(members)
    where = small.where(st.isin([0, 127]))
    where_members = np.nonzero(np.isin(status, [0, 127]))[0]
    _, ids, n_groups = shapes(len(small), 5)[5]
    g = small.groups(ids, n_groups)
    try:
        for sort in SORTS:
            m = F.Matcher("deadbeef", cfg(sort, 1))
            into = m.match_list_into_array(small).copy()
            in_sub, in_where = into[np.isin(into["index"], members)], into[np.isin(into["index"], where_members)]
            for order in ORDERS:
                for pg in (1, 3, None):
                    for s, rows in ((None, into), (sub, in_sub), (where, in_where)):
                        for b, bv in ((None, None), (boost, bvals)):
                            check(m, small, attr, values, order, g, ids, pg, (0, 7, "C", None), rows, subset=s, boost=b,
                                  boost_values=bv, ctx=(sort.name, s is not None, b is not None))
            m.close()
    finally:
        for h in (g, where, sub, boost, st, attr):
            h.close()


def test_latest_row_of_each_group(small):
    """The empty matcher lists every live row: at per_group 1 under ATTR_DESC over a timestamp, the call is each group's
    newest row, newest first (the default screen of a shell-history search), under every strategy."""
    rng = np.random.default_rng(8)
    n = len(small)
    ts = attr_values("timestamps", n, rng)
    attr = small.attr(ts)
    group_of = rng.integers(0, 300, n).astype(np.uint32)
    g = small.groups(group_of, 300)
    newest = {}
    for i in range(n):   # the largest timestamp (timestamps are distinct)
        gi = int(group_of[i])
        if gi not in newest or ts[i] > ts[newest[gi]]:
            newest[gi] = i
    want_index = sorted(newest.values(), key=lambda i: -ts[i])
    try:
        for sort in SORTS:
            m = F.Matcher.from_query("", cfg(sort, 0))
            got, total, counts = m.match_list_ordered_array(small, attr, Order.AttrDesc, 20, groups=g, counts=True)
            assert total == len(newest) and got["index"].tolist() == want_index[:20], sort
            assert counts.tolist() == np.bincount(group_of, minlength=300).tolist()
            check(m, small, attr, ts, Order.AttrDesc, g, group_of, 1, (1, 20, None), m.match_list_into_array(small).copy(),
                  ctx=(sort.name,))
            m.close()
    finally:
        g.close()
        attr.close()


@pytest.mark.parametrize("name", ["multi", "unicode", "long"])
def test_needle_classes(small, name):
    """A multi-pattern query with a negated atom, a unicode needle and a 200-byte needle."""
    rng = np.random.default_rng(9)
    values = attr_values("nulls", len(small), rng)
    attr = small.attr(values)
    _, ids, n_groups = shapes(len(small), 9)[3]
    g = small.groups(ids, n_groups)
    make = {"multi": lambda s: F.Matcher.from_query("dead !^foo", cfg(s, 0)),
            "unicode": lambda s: F.Matcher("é다😀", cfg(s, 1)),
            "long": lambda s: F.Matcher(LONG300[:200], cfg(s, 2))}[name]
    try:
        for sort in SORTS:
            m = make(sort)
            into = m.match_list_into_array(small).copy()
            assert len(into) > 0, name
            for order in ORDERS:
                for pg in (1, 2, None):
                    check(m, small, attr, values, order, g, ids, pg, (1, 7, None), into, ctx=(name, sort.name))
            m.close()
    finally:
        g.close()
        attr.close()


def test_across_edits():
    """Remove, replace, append, then Attr.set and Groups.set."""
    corpus = F.Corpus.from_list(gen(3 * TILE + 100, 31))
    rng = np.random.default_rng(32)
    values = attr_values("nulls", len(corpus), rng)
    ids = rng.integers(0, 30, len(corpus)).astype(np.uint32)
    attr, g = corpus.attr(values), corpus.groups(ids, 30)
    m = F.Matcher("deadbeef", cfg(SortStrategy.ScoreThenIndexDesc, 1))
    try:
        for step in range(5):
            if step == 1:
                got, _ = m.match_list_ordered_array(corpus, attr, Order.AttrDesc, 5, groups=g)
                corpus.remove(got["index"][:2])
                corpus.replace_list(np.array([3, len(corpus) - 1], np.uint32), [b"deadbeef!", b"xdeadbeef"])
            elif step == 2:
                corpus.append_list(gen(700, 33))   # appended rows are null and in no group
                values = np.concatenate([values, np.full(700, ATTR_NULL, np.int64)])
            elif step == 3:
                which = np.array([0, 3, len(corpus) - 1, len(corpus) - 2], np.uint32)
                vals = np.array([I64_MAX, ATTR_NULL, -7, 10**12], np.int64)
                attr.set(which, vals)
                values[which] = vals
            elif step == 4:
                which = np.array([1, 3, len(corpus) - 1, len(corpus) - 5], np.uint32)
                new = np.array([GROUP_NONE, 29, 0, 0], np.uint32)
                g.set(which, new)
                ids = np.concatenate([ids, np.full(len(corpus) - len(ids), GROUP_NONE, np.uint32)])
                ids[which] = new
            into = m.match_list_into_array(corpus).copy()
            for order in ORDERS:
                for pg in (1, 3):
                    check(m, corpus, attr, values, order, g, ids, pg, (3, None), into, ctx=(step,))
    finally:
        m.close()
        g.close()
        attr.close()
        corpus.close()


def test_uncapped_equals_the_ordered_call(small):
    """per_group = UINT64_MAX returns frz_match_list_ordered's rows and total, plus the counts."""
    rng = np.random.default_rng(21)
    values = attr_values("ties", len(small), rng)
    attr = small.attr(values)
    boost = small.boost(rng.integers(-300, 301, len(small)).astype(np.int16))
    _, ids, n_groups = shapes(len(small), 4)[3]
    g = small.groups(ids, n_groups)
    try:
        for sort in SORTS:
            m = F.Matcher("deadbeef", cfg(sort, 1))
            for order in ORDERS:
                for k in (10, None):
                    for b in (None, boost):
                        got, total = m.match_list_ordered_array(small, attr, order, k, boost=b, groups=g, per_group=None)
                        want, wtotal = m.match_list_ordered_array(small, attr, order, k, boost=b)
                        assert total == wtotal
                        expect(got, want, (sort, order, k))
            m.close()
    finally:
        for h in (g, boost, attr):
            h.close()


def test_selection_sizes_at_a_million_rows():
    """|C| just below, at and above the one-block sort's 4096 rows (groups of index % 4095, % 4096, % 4097 at per_group
    1), and k on both sides of it over a larger C."""
    from frizbee_b200 import synth
    data, off = synth.generate("deadbeef", 1 << 20, 48, 64)
    corpus = F.Corpus.from_arrow(data, off)
    rng = np.random.default_rng(13)
    n = len(corpus)
    try:
        values = attr_values("timestamps", n, rng)
        attr = corpus.attr(values)
        for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexDesc):
            m = F.Matcher("deadbeef", cfg(sort, 1))
            into = m.match_list_into_array(corpus).copy()
            assert len(into) > 8 * BLOCK_ROWS
            for mod in (BLOCK_ROWS - 1, BLOCK_ROWS, BLOCK_ROWS + 1):
                ids = (np.arange(n) % mod).astype(np.uint32)
                g = corpus.groups(ids, mod)
                for order in (Order.AttrDesc, Order.ScoreThenAttrAsc):
                    want = check(m, corpus, attr, values, order, g, ids, 1, (50, None), into, ctx=(sort.name, mod))
                    assert len(want) == mod
                g.close()
            ids = (np.arange(n) % 20_000).astype(np.uint32)
            g = corpus.groups(ids, 20_000)
            for order in ORDERS:
                check(m, corpus, attr, values, order, g, ids, 2, (50, BLOCK_ROWS, BLOCK_ROWS + 1, None), into, ctx=(sort.name,))
            g.close()
            m.close()
        attr.close()
    finally:
        corpus.close()


@pytest.mark.parametrize("name", SO.SUBSET_CASES)
def test_survivor_overflow_retry(name):
    lanes = F.Matcher("abcd", Config())
    c = SO.Case(name, lanes.backend_info()["prefilter_lanes"])
    lanes.close()
    sort = SO.SORTS[SO.SUBSET_CASES.index(name)]
    rng = np.random.default_rng(7)
    values = attr_values("timestamps", c.n, rng)
    ids = rng.integers(0, 5000, c.n).astype(np.uint32)
    attr, g = c.corpus.attr(values), c.corpus.groups(ids, 5000)
    m = c.matcher(sort)
    try:
        SO.check_case_overflows(c)
        want, wcounts = specification(c.into, values, Order.AttrDesc, SortStrategy(sort).is_reversed(), ids, 1, 5000)
        # the first call overflows its survivor lists and runs the pipeline again; the collapse and the ordering run once,
        # after the list's length is read back, so the second call launches more than half as many kernels
        got, total, counts = m.match_list_ordered_array(c.corpus, attr, Order.AttrDesc, groups=g, counts=True)
        l1 = m.last_timings()["launches"]
        again, _ = m.match_list_ordered_array(c.corpus, attr, Order.AttrDesc, groups=g)
        l2 = m.last_timings()["launches"]
        assert l2 < l1 < 2 * l2, (name, l1, l2)
        expect(again, got)
        assert total == len(want) and np.array_equal(counts, wcounts)
        expect(got, want)
        got, _ = m.match_list_ordered_array(c.corpus, attr, Order.AttrDesc, 50, groups=g)
        expect(got, want[:50])
    finally:
        m.close()
        g.close()
        attr.close()
        c.corpus.close()


def test_ordered_collapsed_memory(small):
    """Repeated calls at a fixed size (one-block and multi-block sorts, several per_group) hold no more than the first."""
    rng = np.random.default_rng(42)
    attr = small.attr(attr_values("timestamps", len(small), rng))
    boost = small.boost(rng.integers(-300, 301, len(small)).astype(np.int16))
    _, ids, n_groups = shapes(len(small), 6)[3]
    g = small.groups(ids, n_groups)
    m = F.Matcher("deadbeef", cfg(SortStrategy.ScoreThenIndexAsc, 1))
    sub = small.subset(np.arange(0, len(small), 3))

    def calls():
        for order in ORDERS:
            for pg in (1, 32):
                m.match_list_ordered_array(small, attr, order, 10, groups=g, per_group=pg)
                m.match_list_ordered_array(small, attr, order, 10, boost=boost, subset=sub, groups=g, per_group=pg)
                m.match_list_ordered_array(small, attr, order, groups=g, per_group=pg, counts=True)
    try:
        calls()
        held = device_bytes()
        for _ in range(10):
            calls()
        assert device_bytes() == held
    finally:
        for h in (sub, g, boost, attr):
            h.close()
        m.close()


def test_refused_calls(small):
    other = F.Corpus.from_list([b"deadbeef"])
    a_other, g_other = other.attr([1]), other.groups([0], 1)
    attr, g = small.attr([1, 2, 3]), small.groups([0, 0, 1], 2)
    m = F.Matcher("deadbeef", cfg(SortStrategy.ScoreThenIndexAsc, 1))
    try:
        for kw, status in ((dict(attr=a_other, groups=g), 1), (dict(attr=attr, groups=g_other), 1),
                           (dict(attr=attr, groups=g, per_group=0), 1), (dict(attr=attr, groups=g, per_group=33), 9),
                           (dict(attr=attr, groups=g, order=4), 1)):
            with pytest.raises(F.FrizbeeError) as e:
                m.match_list_ordered_array(small, **kw)
            assert e.value.status == status, kw
        values = np.full(len(small), ATTR_NULL, np.int64)
        values[:3] = [1, 2, 3]
        ids = np.full(len(small), GROUP_NONE, np.uint32)
        ids[:3] = [0, 0, 1]
        into = m.match_list_into_array(small).copy()
        check(m, small, attr, values, Order.AttrAsc, g, ids, 1, (9,), into)   # a refused call leaves nothing behind
    finally:
        m.close()
        for h in (g, attr, g_other, a_other):
            h.close()
        other.close()
