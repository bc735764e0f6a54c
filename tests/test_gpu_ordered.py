"""Ordered calls on the GPU (frz_match_list_ordered).  The contract: the rows of match_list_into (or of a subset's
members), reversed for the *_DESC strategies, sorted stably by tests/ordering.py's order_by_attr (the attribute, nulls
last, and clamp(score + boost[index], 0, 65535) or the raw score), truncated to the first k; the reported total is the
full count.  Every check compares bit for bit with order_by_attr applied to the GPU's own match_list_into (pinned to the
oracle by the parity tests): every order and strategy, subsets and boosts, attribute shapes, corpus edits, the empty
matcher and every needle class, selections on both sides of the one-block sort, the survivor-overflow retry, against the
ranked and top-K calls, and for the device memory the calls hold."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
import test_gpu_survivor_overflow as SO
from frizbee_b200.types import Config, Order, SortStrategy
from ordering import ATTR_NULL, order_by_attr
from test_gpu_ranked import LONG300, gen

pytestmark = pytest.mark.gpu

TILE = 1024
LANES = 32
BLOCK_ROWS = 4096   # kFrzOrderBlockRows: larger selections take the multi-block sort
I64_MAX = 2**63 - 1
ORDERS = list(Order)
SORTS = list(SortStrategy)


def cfg(sort, max_typos=0, **kw):
    return Config(max_typos=max_typos, sort=sort, emulate_lanes=LANES, **kw)


def expect(got, want, ctx=()):
    assert len(got) == len(want), (ctx, len(got), len(want))
    for f in ("index", "score", "exact"):
        bad = np.nonzero(got[f] != want[f])[0]
        assert bad.size == 0, (ctx, f, bad[:5], got[bad[:5]], want[bad[:5]])


def attr_values(kind, n, rng):
    if kind == "nulls":
        v = rng.integers(-1000, 1000, n).astype(np.int64)
        v[rng.random(n) < 0.3] = ATTR_NULL
    elif kind == "ties":
        v = rng.choice([0, 1, 127], n).astype(np.int64)
    elif kind == "timestamps":
        v = 1_600_000_000_000 + rng.permutation(n).astype(np.int64) * 7
    elif kind == "extremes":
        v = rng.choice([ATTR_NULL, ATTR_NULL + 1, ATTR_NULL + 2, -1, 0, 1, I64_MAX - 1, I64_MAX], n).astype(np.int64)
    elif kind == "short":   # an attribute shorter than the corpus
        v = rng.integers(-5, 5, n // 3).astype(np.int64)
    else:
        raise ValueError(kind)
    return v


def check(m, corpus, attr, values, order, k, subset=None, boost=None, boost_values=None, rows=None, ctx=()):
    """One ordered call against order_by_attr over the GPU's own match_list_into (rows: that list, restricted to the
    subset's members when there is one)."""
    if rows is None:
        rows = m.match_list_into_array(corpus).copy()
    want = order_by_attr(rows, values, int(order), SortStrategy(m.config.sort).is_reversed(), boost_values)
    got, total = m.match_list_ordered_array(corpus, attr, order, k, subset=subset, boost=boost)
    assert total == len(want), (ctx, total, len(want))
    expect(got, want if k is None else want[:k], ctx)
    return want


@pytest.fixture(scope="module")
def small():
    corpus = F.Corpus.from_list(gen(6 * TILE + 321, 11))
    yield corpus
    corpus.close()


@pytest.mark.parametrize("kind", ["nulls", "ties", "timestamps", "extremes", "short"])
def test_orders_strategies_and_k(small, kind):
    rng = np.random.default_rng(["nulls", "ties", "timestamps", "extremes", "short"].index(kind))
    values = attr_values(kind, len(small), rng)
    attr = small.attr(values)
    bvals = rng.integers(-300, 301, len(small)).astype(np.int16)
    boost = small.boost(bvals)
    members = np.sort(rng.choice(len(small), len(small) // 3, replace=False)).astype(np.uint32)
    sub = small.subset(members)
    try:
        for sort in SORTS:
            m = F.Matcher("deadbeef", cfg(sort, 1))
            try:
                into = m.match_list_into_array(small).copy()
                into_sub = into[np.isin(into["index"], members)]
                n = len(into)
                for order in ORDERS:
                    for k in (0, 1, 7, n, n + 5, None):
                        check(m, small, attr, values, order, k, rows=into, ctx=(kind, sort, order, k))
                    for b, bv in ((boost, bvals), (None, None)):
                        for k in (7, None):
                            check(m, small, attr, values, order, k, subset=sub, boost=b, boost_values=bv, rows=into_sub,
                                  ctx=(kind, sort, order, k, "subset", b is not None))
                        check(m, small, attr, values, order, 7, boost=b, boost_values=bv, rows=into,
                              ctx=(kind, sort, order, "boost", b is not None))
            finally:
                m.close()
    finally:
        sub.close()
        boost.close()
        attr.close()


def test_where_subset(small):
    rng = np.random.default_rng(5)
    values = attr_values("ties", len(small), rng)
    ts = attr_values("timestamps", len(small), rng)
    status, stamp = small.attr(values), small.attr(ts)
    sub = small.where(status.isin([0, 127]))
    members = np.nonzero(np.isin(values, [0, 127]))[0]
    try:
        for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexDesc):
            m = F.Matcher("deadbeef", cfg(sort, 1))
            into = m.match_list_into_array(small).copy()
            rows = into[np.isin(into["index"], members)]
            for order in ORDERS:
                for k in (50, None):
                    check(m, small, stamp, ts, order, k, subset=sub, rows=rows, ctx=(sort, order, k))
            m.close()
    finally:
        sub.close()
        status.close()
        stamp.close()


@pytest.mark.parametrize("name", ["empty", "multi", "unicode", "long"])
def test_needle_classes(small, name):
    rng = np.random.default_rng(9)
    values = attr_values("nulls", len(small), rng)
    attr = small.attr(values)
    make = {"empty": lambda s: F.Matcher.from_query("", cfg(s, 0)),
            "multi": lambda s: F.Matcher.from_query("dead beef", cfg(s, 0)),
            "unicode": lambda s: F.Matcher("é다😀", cfg(s, 1)),
            "long": lambda s: F.Matcher(LONG300[:200], cfg(s, 2))}[name]
    try:
        for sort in SORTS:
            m = make(sort)
            into = m.match_list_into_array(small).copy()
            assert len(into) > 0, name
            for order in ORDERS:
                for k in (1, 7, None):
                    check(m, small, attr, values, order, k, rows=into, ctx=(name, sort, order, k))
            m.close()
    finally:
        attr.close()


def test_selection_sizes_at_a_million_rows():
    """k = 50 (one-block sort), a k just above the block's capacity (exact select, multi-block sort) and the whole list,
    for a high-cardinality and a tie-heavy attribute."""
    from frizbee_b200 import synth
    data, off = synth.generate("deadbeef", 1 << 20, 48, 64)
    corpus = F.Corpus.from_arrow(data, off)
    rng = np.random.default_rng(13)
    try:
        for kind in ("timestamps", "ties"):
            values = attr_values(kind, len(corpus), rng)
            attr = corpus.attr(values)
            for sort in (SortStrategy.ScoreThenIndexAsc, SortStrategy.IndexDesc):
                m = F.Matcher("deadbeef", cfg(sort, 1))
                into = m.match_list_into_array(corpus).copy()
                assert len(into) > 4 * BLOCK_ROWS
                for order in ORDERS:
                    for k in (50, BLOCK_ROWS, BLOCK_ROWS + 1, None):
                        check(m, corpus, attr, values, order, k, rows=into, ctx=(kind, sort, order, k))
                m.close()
            attr.close()
    finally:
        corpus.close()


def test_across_edits():
    corpus = F.Corpus.from_list(gen(3 * TILE + 100, 31))
    rng = np.random.default_rng(32)
    values = attr_values("nulls", len(corpus), rng)
    attr = corpus.attr(values)
    m = F.Matcher("deadbeef", cfg(SortStrategy.ScoreThenIndexDesc, 1))
    try:
        for step in range(4):
            if step == 1:
                corpus.append_list(gen(700, 33))   # appended rows are null
                values = np.concatenate([values, np.full(700, ATTR_NULL, np.int64)])
            elif step == 2:
                got, _ = m.match_list_ordered_array(corpus, attr, Order.AttrDesc, 5)
                corpus.remove(got["index"][:2])
                corpus.replace_list(np.array([3, len(corpus) - 1], np.uint32), [b"deadbeef!", b"xdeadbeef"])
            elif step == 3:
                which = np.array([0, 3, len(corpus) - 1, len(corpus) - 2], np.uint32)
                vals = np.array([I64_MAX, ATTR_NULL, -7, 10**12], np.int64)
                attr.set(which, vals)
                values[which] = vals
            for order in ORDERS:
                for k in (3, None):
                    check(m, corpus, attr, values, order, k, ctx=(step, order, k))
    finally:
        m.close()
        attr.close()
        corpus.close()


def test_against_ranked_and_top(small):
    """An all-null attribute orders by score (with the boost) alone: SCORE_THEN_ATTR_* equals the ranked call with the same
    boost (an all-zero one without), and, without a boost under a by-score strategy, the top-K call.  The row index as the
    attribute under ATTR_ASC, without a boost and under an unreversed strategy, is index order."""
    rng = np.random.default_rng(21)
    null = small.attr()
    index = small.attr(np.arange(len(small), dtype=np.int64))
    bvals = rng.integers(-300, 301, len(small)).astype(np.int16)
    boost, zero = small.boost(bvals), small.boost()
    try:
        for sort in SORTS:
            m = F.Matcher("deadbeef", cfg(sort, 1))
            for order in (Order.ScoreThenAttrDesc, Order.ScoreThenAttrAsc):
                for k in (10, None):
                    for b in (boost, None):
                        got, total = m.match_list_ordered_array(small, null, order, k, boost=b)
                        want, wtotal = m.match_list_ranked_array(small, b if b is not None else zero, k)
                        assert total == wtotal
                        expect(got, want, (sort, order, k))
                    if SortStrategy(sort) in (SortStrategy.ScoreThenIndexAsc, SortStrategy.ScoreThenIndexDesc):
                        got, total = m.match_list_ordered_array(small, null, order, k)
                        want, wtotal = m.match_list_top_array(small, k if k is not None else len(small))
                        assert total == wtotal
                        expect(got, want, (sort, order, k, "top"))
            if not SortStrategy(sort).is_reversed():
                got, _ = m.match_list_ordered_array(small, index, Order.AttrAsc)
                expect(got, m.match_list_into_array(small), sort)
            m.close()
    finally:
        for h in (null, index, boost, zero):
            h.close()


@pytest.fixture(scope="module")
def lanes():
    m = F.Matcher("abcd", Config())
    try:
        return m.backend_info()["prefilter_lanes"]
    finally:
        m.close()


@pytest.mark.parametrize("name", SO.SUBSET_CASES)
def test_survivor_overflow_retry(lanes, name):
    c = SO.Case(name, lanes)
    sort = SO.SORTS[SO.SUBSET_CASES.index(name)]
    rng = np.random.default_rng(7)
    values = attr_values("ties", c.n, rng)
    attr = c.corpus.attr(values)
    m = c.matcher(sort)
    try:
        SO.check_case_overflows(c)
        want = order_by_attr(c.into, values, int(Order.AttrDesc), SortStrategy(sort).is_reversed())
        # the first call overflows its survivor lists and runs the pipeline again; the ordering runs once, after the
        # list's length is read back, so the second call launches more than half as many kernels
        got, total = m.match_list_ordered_array(c.corpus, attr, Order.AttrDesc)
        l1 = m.last_timings()["launches"]
        again, _ = m.match_list_ordered_array(c.corpus, attr, Order.AttrDesc)
        l2 = m.last_timings()["launches"]
        assert l2 < l1 < 2 * l2, (name, l1, l2)
        expect(again, got)
        assert total == len(want)
        expect(got, want)
        got, total = m.match_list_ordered_array(c.corpus, attr, Order.AttrDesc, 50)
        expect(got, want[:50])
    finally:
        m.close()
        attr.close()
        c.corpus.close()


def device_bytes():
    L = F.lib()
    L.frz_debug_device_bytes.restype = C.c_uint64
    L.frz_debug_device_bytes.argtypes = []
    return L.frz_debug_device_bytes()


def test_ordered_memory(small):
    """Repeated ordered calls at a fixed size (one-block and multi-block sorts, with and without a select) hold no more
    than the first."""
    rng = np.random.default_rng(42)
    attr = small.attr(attr_values("timestamps", len(small), rng))
    boost = small.boost(rng.integers(-300, 301, len(small)).astype(np.int16))
    m = F.Matcher("deadbeef", cfg(SortStrategy.ScoreThenIndexAsc, 1))
    sub = small.subset(np.arange(0, len(small), 3))

    def calls():
        for order in ORDERS:
            m.match_list_ordered_array(small, attr, order, 10)
            m.match_list_ordered_array(small, attr, order, 10, boost=boost, subset=sub)
            m.match_list_ordered_array(small, attr, order)
    try:
        calls()
        held = device_bytes()
        for _ in range(10):
            calls()
        assert device_bytes() == held
    finally:
        sub.close()
        m.close()
        boost.close()
        attr.close()


def test_refused_calls(small):
    other = F.Corpus.from_list([b"deadbeef"])
    a_other = other.attr([1])
    attr = small.attr([1, 2, 3])
    m = F.Matcher("deadbeef", cfg(SortStrategy.ScoreThenIndexAsc, 1))
    try:
        with pytest.raises(F.FrizbeeError) as e:
            m.match_list_ordered_array(small, a_other)
        assert e.value.status == 1
        with pytest.raises(F.FrizbeeError) as e:
            m.match_list_ordered_array(small, attr, 4)
        assert e.value.status == 1
        values = np.full(len(small), ATTR_NULL, np.int64)
        values[:3] = [1, 2, 3]
        check(m, small, attr, values, Order.AttrAsc, 9)   # a refused call leaves nothing behind
    finally:
        m.close()
        attr.close()
        a_other.close()
        other.close()
