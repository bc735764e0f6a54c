"""Subsets filled from attributes on the GPU (frz_attr_*, frz_subset_where).  The contract: a filled subset behaves bit for
bit like frz_subset_create over the indices the clauses select.  Every filled subset is checked against
corpus.subset(np.flatnonzero(mask)), mask being a numpy restatement of the clauses: equal len(), and equal results from the
subset, top-K, ranked, collapsed, column and batched calls, for corpus lengths around word, chunk and tile boundaries up to
10 M rows, random conjunctions of 0-8 clauses at densities from empty to full, and bases (including the subset itself and
a base made before an append).  Also: corpus edits after the attribute was made, refills and device memory, and refused
calls.  Needs a CUDA device."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200 import synth
from frizbee_b200.types import Config, SortStrategy

pytestmark = pytest.mark.gpu

NULL = F.ATTR_NULL
I64_MAX = 2**63 - 1
WORDS = [b"foo", b"fooBar", b"foo_bar", b"barfoo", b"deadbeef", b"dbf", "é다x".encode(), b"src/matcher/mod.rs", b"",
         b"needle in a haystack", b"a" * 70 + b"deadbeef", b"bar"]
LONG = "a" * 66 + "dead"   # a 70-byte needle


def rows(n, seed):
    """Arrow buffers of n rows: short words for small n, the synthetic flagship shape from 100 k rows up."""
    if n >= 100_000:
        return synth.generate("deadbeef", n, 24, 64, seed)
    rng = np.random.default_rng(seed)
    return F.pack_host([WORDS[int(i)] + WORDS[int(j)] for i, j in rng.integers(0, len(WORDS), (n, 2))])


def matchers(sort):
    """The empty matcher, a short fuzzy byte needle, a unicode needle, a 70-byte needle and a multi-pattern query with a
    negated atom."""
    cfg = Config(max_typos=1, sort=sort)
    return [F.Matcher.from_query("", cfg), F.Matcher("dbf", cfg), F.Matcher("é다", cfg), F.Matcher(LONG, cfg.with_(max_typos=2)),
            F.Matcher.from_query("foo !^bar", cfg)]


ALL_MATCHERS = {s: matchers(s) for s in SortStrategy}


def attr_values(n, rng):
    """Three columns: a timestamp, a skewed directory id and an exit status, with nulls, extremes and short arrays (the rows
    past an attribute's array are null)."""
    ts = rng.integers(0, 1_000_000, n).astype(np.int64)
    d = np.minimum(rng.zipf(1.3, n), 10_000).astype(np.int64)
    ex = np.where(rng.random(n) < 0.8, 0, rng.integers(-3, 130, n)).astype(np.int64)
    for v in (ts, d, ex):
        v[rng.random(n) < 0.05] = NULL
        k = min(n, 4)
        v[:k] = np.array([NULL + 1, I64_MAX, -1, 0])[:k]
    lens = [n, n - min(n, int(rng.integers(0, 40))), n]
    return [v[:m].copy() for v, m in zip((ts, d, ex), lens)]


def full(values, n):
    out = np.full(n, NULL, np.int64)
    out[: len(values)] = values
    return out


def spec(values, lo=0, hi=-1, in_=None, negate=False):
    t = np.isin(values, np.asarray(in_, np.int64)) if in_ is not None else (lo <= values) & (values <= hi)
    return (t != negate) & (values != NULL)


def random_clauses(attrs, vals, n, rng, n_clauses=None, density=None):
    """(clauses, mask): 0-8 random range, equality and set clauses, some negated.  density 'sparse' (an equality on the
    timestamp) or 'dense' (exit status not 77) picks the first clause."""
    k = int(rng.integers(0, 9)) if n_clauses is None else n_clauses
    cols = {id(a): full(v, n) for a, v in zip(attrs, vals)}
    out, mask = [], np.ones(n, bool)
    for j in range(k):
        a = int(rng.integers(0, 3))
        real = cols[id(attrs[a])][cols[id(attrs[a])] != NULL]
        pick = lambda: int(rng.choice(real)) if real.size else 0
        kind = int(rng.integers(0, 4))
        if j == 0 and density == "sparse":
            ts = cols[id(attrs[0])]
            x = int(rng.choice(ts[ts != NULL])) if (ts != NULL).any() else 0
            w = attrs[0].between(x, x)
        elif j == 0 and density == "dense":
            w = ~attrs[2].isin([77])
        elif kind == 0:
            lo, hi = sorted([pick(), pick()])
            w = attrs[a].between(lo, hi)
        elif kind == 1:
            x = pick()
            w = attrs[a].between(x, x)
        elif kind == 2:
            w = attrs[a].isin([pick() for _ in range(int(rng.integers(1, 21)))] + [12345678])
        else:
            w = attrs[a].between(pick(), pick())   # maybe lo > hi: holds for no value
        if rng.random() < 0.25 and not (j == 0 and density):
            w = ~w
        out.append(w)
        mask &= spec(cols[id(w.attr)], w.lo, w.hi, w.values, w.negate)
    return out, mask


def assert_same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), what


def check(corpus, filled, mask, what, heavy=True, sorts=tuple(SortStrategy)):
    """filled behaves as frz_subset_create over np.flatnonzero(mask) in every call that takes a subset."""
    ref = corpus.subset(np.flatnonzero(mask))
    try:
        assert len(filled) == len(ref) == int(mask.sum()), what
        for s in sorts:
            for m in ALL_MATCHERS[s] if heavy else ALL_MATCHERS[s][:2]:
                assert_same(m.match_list_subset_array(corpus, filled), m.match_list_subset_array(corpus, ref), (what, s, "list"))
                a, ta = m.match_list_subset_top_array(corpus, filled, 7)
                b, tb = m.match_list_subset_top_array(corpus, ref, 7)
                assert ta == tb, (what, s)
                assert_same(a, b, (what, s, "top"))
        if not heavy:
            return
        rng = np.random.default_rng(len(corpus))
        m = ALL_MATCHERS[SortStrategy.ScoreThenIndexAsc][1]
        boost = corpus.boost(rng.integers(-300, 300, len(corpus)).astype(np.int16))
        groups = corpus.groups(rng.integers(0, 17, len(corpus)).astype(np.uint32), 17)
        try:
            a, ta = m.match_list_ranked_array(corpus, boost, 20, filled)
            b, tb = m.match_list_ranked_array(corpus, boost, 20, ref)
            assert ta == tb and np.array_equal(a, b), (what, "ranked")
            a = m.match_list_collapsed_array(corpus, groups, 20, 2, filled, boost, counts=True)
            b = m.match_list_collapsed_array(corpus, groups, 20, 2, ref, boost, counts=True)
            assert a[1] == b[1] and np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2]), (what, "collapsed")
            ms = [m, ALL_MATCHERS[SortStrategy.ScoreThenIndexAsc][4]]
            a = F.match_list_columns(ms, [corpus, corpus], 20, subset=filled, groups=groups, counts=True)
            b = F.match_list_columns(ms, [corpus, corpus], 20, subset=ref, groups=groups, counts=True)
            assert a[1] == b[1] and np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2]), (what, "columns")
        finally:
            boost.close()
            groups.close()
    finally:
        ref.close()


BATCH_NEEDLES = ["foo", "bar", "dbf", "dead", "beef", "fooBar", "src", "mod", "needle", "hay", "oo", "ar"]


def check_batch(corpus, filled, mask):
    """match_list_batch over 40 batched-class queries, half of them scoped to the filled subset, equals the same batch
    scoped to frz_subset_create's subset, and ran the batched kernels."""
    ref = corpus.subset(np.flatnonzero(mask))
    try:
        ms = [F.Matcher(BATCH_NEEDLES[j % len(BATCH_NEEDLES)], Config(max_typos=0, sort=SortStrategy(j % 4))) for j in range(40)]
        a = F.match_list_batch(ms, corpus, 10, subsets=[filled if j % 2 else None for j in range(40)])
        assert F.batch_last()["sub_batches"] > 0
        b = F.match_list_batch(ms, corpus, 10, subsets=[ref if j % 2 else None for j in range(40)])
        for x, y in zip(a, b):
            assert np.array_equal(x, y)
    finally:
        ref.close()


def new_corpus(n, seed):
    data, off = rows(n, seed)
    return F.Corpus.from_arrow(data, off)


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 1023, 1024, 1025, 3 * 1024 + 7, 100_000, 1_000_000])
def test_fill_equals_create(n):
    rng = np.random.default_rng(n + 7)
    corpus = new_corpus(n, n)
    vals = attr_values(n, rng)
    attrs = [corpus.attr(v) for v in vals]
    s = corpus.subset([])
    heavy = n <= 100_000
    try:
        cases = [(None, 0), ("sparse", None), ("dense", None), (None, None), (None, 8), ("sparse", 3), (None, 1)]
        for trial, (density, k) in enumerate(cases):
            cl, mask = random_clauses(attrs, vals, n, rng, k, density)
            s.where(*cl)
            check(corpus, s, mask, (n, trial), heavy=heavy)
            fresh = corpus.where(*cl)
            check(corpus, fresh, mask, (n, trial, "fresh"), heavy=False, sorts=(SortStrategy.IndexAsc,))
            # with a base: another subset, then the subset itself (refining in place)
            cl2, mask2 = random_clauses(attrs, vals, n, rng, int(rng.integers(0, 4)))
            s.where(*cl2, base=fresh)
            check(corpus, s, mask & mask2, (n, trial, "base"), heavy=heavy and trial < 2)
            cl3, mask3 = random_clauses(attrs, vals, n, rng, int(rng.integers(0, 3)))
            s.where(*cl3, base=s)
            check(corpus, s, mask & mask2 & mask3, (n, trial, "base=self"), heavy=False)
            if n in (33, 3 * 1024 + 7, 100_000) and trial in (1, 2):
                check_batch(corpus, s, mask & mask2 & mask3)
            fresh.close()
        assert len(s.where()) == n and len(s.where(base=corpus.subset([]))) == 0
    finally:
        s.close()
        for a in attrs:
            a.close()
        corpus.close()


def test_ten_million_rows():
    n = 10_000_000   # about 9 800 scan chunks
    rng = np.random.default_rng(10)
    corpus = new_corpus(n, 10)
    vals = attr_values(n, rng)
    attrs = [corpus.attr(v) for v in vals]
    s = corpus.subset([])
    try:
        for density, k in (("sparse", 2), ("dense", 1), (None, 8), (None, 0)):
            cl, mask = random_clauses(attrs, vals, n, rng, k, density)
            s.where(*cl)
            check(corpus, s, mask, (n, density, k), heavy=False, sorts=(SortStrategy.IndexAsc, SortStrategy.ScoreThenIndexAsc))
    finally:
        s.close()
        for a in attrs:
            a.close()
        corpus.close()


def test_edits_after_the_attribute():
    n = 5000
    corpus = new_corpus(n, 3)
    rng = np.random.default_rng(3)
    v = rng.integers(0, 10, n).astype(np.int64)
    a = corpus.attr(v)
    old = corpus.where(a.between(0, 4))               # a base made before the append
    removed = rng.choice(n, 300, replace=False)
    replaced = rng.choice(n, 200, replace=False)
    corpus.remove(removed)
    corpus.replace_list(replaced, [b"deadbeef dbf foo" for _ in replaced])
    corpus.append_list([b"dbf appended"] * 1500)
    m = n + 1500
    s = corpus.where(a.between(0, 4))
    vf = full(v, m)                                    # appended rows are null until set
    check(corpus, s, spec(vf, 0, 4), "edited")
    check(corpus, corpus.where(~a.between(0, 4)), spec(vf, 0, 4, negate=True), "edited, negated")
    assert len(corpus.where()) == m                    # no clause: every row, removed ones counted
    new_idx = np.arange(n, m, 3, dtype=np.uint32)
    a.set(new_idx, np.full(len(new_idx), 2, np.int64))
    a.set(np.arange(0, 100, dtype=np.uint32), np.full(100, NULL, np.int64))   # FRZ_ATTR_NULL clears a value
    vf[new_idx] = 2
    vf[:100] = NULL
    s.where(a.between(0, 4))
    check(corpus, s, spec(vf, 0, 4), "set after append")
    s.where(a.isin([2, 3]), base=old)                  # members of the old base only below its length
    base_mask = np.zeros(m, bool)
    base_mask[:n] = spec(full(v, n), 0, 4)
    check(corpus, s, spec(vf, in_=[2, 3]) & base_mask, "old base")
    corpus.append_list([b"foo"] * 40)                  # s's bitmap must grow while it is its own base
    s.where(a.between(2, 2), base=s)
    mf = np.zeros(m + 40, bool)
    mf[:m] = spec(vf, in_=[2, 3]) & base_mask & spec(vf, 2, 2)
    check(corpus, s, mf, "grow in place")
    for h in (s, old):
        h.close()
    a.close()
    corpus.close()


def _bytes():
    L = F.lib()
    L.frz_debug_device_bytes.restype = C.c_uint64
    L.frz_debug_device_bytes.argtypes = []
    return L.frz_debug_device_bytes()


def test_refills_and_device_memory():
    n = 300_000
    corpus = new_corpus(n, 4)
    rng = np.random.default_rng(4)
    v = rng.integers(0, 1000, n).astype(np.int64)
    widths = [0, 1, 10, 100, 500, 1000, 20, 3, 1000, 0, 250]
    start = _bytes()
    a = corpus.attr(v)
    s = corpus.subset([])
    after = []
    for w in widths:   # refills only: the device memory they hold
        s.where(a.between(0, w - 1))
        assert len(s) == int((v < w).sum())
        after.append(_bytes())
    largest = widths.index(1000)
    assert all(x == after[largest] for x in after[largest:]), after   # grow-only: nothing grows after the largest fill
    for w in widths:   # refills at changing densities equal fresh subsets
        extra = [int(x) for x in rng.integers(0, 1000, 300)]
        s.where(a.between(0, w - 1), a.isin(extra))
        check(corpus, s, spec(v, 0, w - 1) & spec(v, in_=extra), ("refill", w), heavy=False, sorts=(SortStrategy.ScoreThenIndexAsc,))
    s.close()
    a.close()
    assert _bytes() == start   # the attribute and the subset held all of it
    corpus.close()


def test_refused_calls():
    c1, c2 = new_corpus(100, 5), new_corpus(100, 6)
    a1, a2 = c1.attr(np.arange(100)), c2.attr(np.arange(100))
    s1, s2 = c1.subset([1, 2, 3]), c2.subset([4])
    with pytest.raises(F.FrizbeeError, match="attribute was made on another corpus"):
        s1.where(a2.between(0, 10))
    with pytest.raises(F.FrizbeeError, match="base subset was made on another corpus"):
        s1.where(a1.between(0, 10), base=s2)
    with pytest.raises(F.FrizbeeError, match="FRZ_ATTR_NULL"):
        s1.where(a1.isin([1, NULL]))
    with pytest.raises(F.FrizbeeError) as e:
        s1.where(*[a1.between(0, 99)] * 9)
    assert e.value.status_name == "FRZ_ERR_UNSUPPORTED"
    assert len(s1) == 3   # a refused call leaves the subset as it was
    m = ALL_MATCHERS[SortStrategy.IndexAsc][0]
    assert list(m.match_list_subset_array(c1, s1)["index"]) == [1, 2, 3]
    for which, vals in (([5, 5], [1, 2]), ([100], [1]), ([3, 200], [1, 2])):
        with pytest.raises(F.FrizbeeError):
            a1.set(which, vals)
    with pytest.raises(F.FrizbeeError):
        c1.attr(np.arange(101))
    s1.where(a1.between(0, 99))
    assert len(s1) == 100   # the refused sets changed nothing
    for h in (s1, s2, a1, a2, c1, c2):
        h.close()
