"""Boosts filled from attribute rules on the GPU (frz_boost_where, frz_boost_where_batch: Boost.where, F.boost_where_batch).
The contract: each boost holds clamp(base + the adds of the rules whose clause holds) per row, and a ranked call over it
is bit for bit the same call over corpus.boost(those values).  Checked against a numpy restatement (Boost.values()), at
corpus lengths around chunk boundaries up to 10 M rows, after corpus edits, in place, through match_list_ranked_array in
every sort strategy with and without a subset and through match_list_batch, at key bounds on both sides of the two-pass
sort, for batched fills against per-query fills, for device memory on refills, and for refused calls.  Needs a CUDA
device."""
import ctypes as C

import numpy as np
import pytest

import frizbee_b200 as F
from frizbee_b200.types import Config, SortStrategy
from test_gpu_where import BATCH_NEEDLES, NULL, attr_values, full, new_corpus, rows, spec

pytestmark = pytest.mark.gpu

STAGED = 4   # kFrzWhereBatchStaged


def random_rules(attrs, vals, n, rng, n_rules=None):
    """Up to 8 rules over the attributes: (BoostRule list, the restated (mask, add) of each)."""
    k = int(rng.integers(0, 9)) if n_rules is None else n_rules
    out, spec_rules = [], []
    for _ in range(k):
        a = int(rng.integers(len(attrs)))
        v = full(vals[a], n)
        pick = v[v != NULL]
        add = int(rng.integers(-65535, 65536)) if rng.random() < 0.2 else int(rng.integers(-200, 201))
        neg = bool(rng.random() < 0.25)
        if rng.random() < 0.6 or pick.size == 0:
            lo, hi = sorted(int(x) for x in rng.choice(pick if pick.size else np.array([0, 5]), 2))
            w = attrs[a].between(lo, hi)
            mask = spec(v, lo, hi, negate=neg)
        else:
            s = rng.choice(pick, int(rng.integers(1, 6)))
            w = attrs[a].isin(s)
            mask = spec(v, in_=s, negate=neg)
        out.append((~w if neg else w).add(add))
        spec_rules.append((mask, add))
    return out, spec_rules


def expected(n, spec_rules, base=None):
    acc = np.zeros(n, np.int64)
    if base is not None:
        acc[: len(base)] += base.astype(np.int64)
    for mask, add in spec_rules:
        acc += np.where(mask, add, 0)
    return np.clip(acc, -32768, 32767).astype(np.int16)


def ranked_equal(corpus, filled, want, subset=None, sorts=tuple(SortStrategy), k=50):
    """match_list_ranked_array over the filled boost equals the call over corpus.boost(want), strategy by strategy."""
    ref = corpus.boost(want)
    try:
        for sort in sorts:
            m = F.Matcher("dbf", Config(max_typos=1, sort=sort))
            a, ta = m.match_list_ranked_array(corpus, filled, k, subset)
            b, tb = m.match_list_ranked_array(corpus, ref, k, subset)
            m.close()
            assert ta == tb and np.array_equal(a, b), sort
    finally:
        ref.close()


@pytest.mark.parametrize("n", [0, 1, 31, 1023, 1024, 1025, 3 * 1024 + 7, 100_000, 1_000_000])
def test_values_equal_numpy(n):
    rng = np.random.default_rng(n + 11)
    corpus = new_corpus(n, n)
    vals = attr_values(n, rng)
    attrs = [corpus.attr(v) for v in vals]
    b = corpus.boost()
    base = corpus.boost(rng.integers(-3000, 3000, n // 2).astype(np.int16))
    host_base = base.values()
    try:
        for trial in range(6):
            rules, sr = random_rules(attrs, vals, n, rng, 8 if trial == 0 else None)
            with_base = trial % 2 == 1
            got = b.where(*rules, base=base if with_base else None).values()
            want = expected(n, sr, host_base if with_base else None)
            assert np.array_equal(got, want), (n, trial)
            if 31 <= n <= 100_000 and trial < 2:
                sub = corpus.subset(np.arange(0, n, 3))
                ranked_equal(corpus, b, want, sorts=tuple(SortStrategy))
                ranked_equal(corpus, b, want, subset=sub, sorts=tuple(SortStrategy))
                sub.close()
        # in place: add to the current values
        before = b.values()
        rules, sr = random_rules(attrs, vals, n, rng, 3)
        assert np.array_equal(b.where(*rules, base=b).values(), expected(n, sr, before))
        # no rules: a copy of the base, or zero
        assert np.array_equal(b.where(base=base).values(), expected(n, [], host_base))
        assert not b.where().values().any()
    finally:
        for h in attrs + [b, base]:
            h.close()
        corpus.close()


def test_ten_million_rows():
    n = 10_000_000
    rng = np.random.default_rng(10)
    corpus = new_corpus(n, 10)
    ts = rng.integers(0, 1_000_000, n).astype(np.int64)
    d = np.minimum(rng.zipf(1.3, n), 10_000).astype(np.int64)
    ta, da = corpus.attr(ts), corpus.attr(d)
    frec = corpus.boost(rng.integers(0, 100, n).astype(np.int16))
    b = corpus.boost()
    try:
        now = 1_000_000
        got = b.where(ta.between(now - 1000, now).add(30), ta.between(now - 10_000, now).add(20),
                      ta.between(now - 100_000, now).add(10), da.isin([1, 7]).add(15), base=frec).values()
        want = frec.values().astype(np.int64) + 15 * np.isin(d, [1, 7])
        want += 30 * (ts >= now - 1000) + 20 * (ts >= now - 10_000) + 10 * (ts >= now - 100_000)
        assert np.array_equal(got, want.astype(np.int16))
        ranked_equal(corpus, b, want.astype(np.int16), sorts=(SortStrategy.ScoreThenIndexAsc,))
    finally:
        for h in (ta, da, frec, b):
            h.close()
        corpus.close()


def test_after_edits():
    n = 5000
    rng = np.random.default_rng(3)
    data, off = rows(n, 3)
    corpus = F.Corpus.from_arrow(data, off)
    vals = attr_values(n, rng)
    attrs = [corpus.attr(v) for v in vals]
    b = corpus.boost(rng.integers(-50, 50, 100).astype(np.int16))
    try:
        rules, sr = random_rules(attrs, vals, n, rng, 5)
        b.where(*rules)
        assert np.array_equal(b.values(), expected(n, sr))
        # rows appended after the fill are 0 until the next fill; the attributes are null there
        corpus.append_list(["deadbeef", "dbf", "foo"])
        assert np.array_equal(b.values(), np.concatenate([expected(n, sr), np.zeros(3, np.int16)]))
        n2 = n + 3
        ext = [(np.concatenate([m, np.zeros(3, bool)]), a) for m, a in sr]
        b.where(*rules)
        first = b.values()
        assert np.array_equal(first, expected(n2, ext))
        # removed rows keep their boost (kept by index); replaced rows too
        corpus.remove([0, 17, 4999])
        corpus.replace_list([5, 6], ["dbfdbf", "x"])
        b.where(*rules, base=b)
        want = expected(n2, ext, first)
        assert np.array_equal(b.values(), want)
        ranked_equal(corpus, b, want)
        # Boost.set works on a filled boost as on any other
        b.set([n2 - 1, 3], [1234, -7])
        want[[n2 - 1, 3]] = [1234, -7]
        assert np.array_equal(b.values(), want)
        ranked_equal(corpus, b, want)
    finally:
        for h in attrs + [b]:
            h.close()
        corpus.close()


def test_key_bound_both_ways():
    """A fill whose maximum lifts the key bound past 1024 (the two-pass sort), then one that lowers it to 0: both rank as a
    boost made from the same values."""
    n = 20_000
    rng = np.random.default_rng(5)
    corpus = new_corpus(n, 5)
    ts = rng.integers(0, 100, n).astype(np.int64)
    a = corpus.attr(ts)
    b = corpus.boost()
    try:
        for rules, spec_rules in (([a.between(0, 9).add(2000), a.between(5, 50).add(-30)], [(ts <= 9, 2000), ((ts >= 5) & (ts <= 50), -30)]),
                                  ([a.between(0, 99).add(-5), (~a.between(0, 9)).add(-1000)], [(ts >= 0, -5), (ts > 9, -1000)])):
            b.where(*rules)
            want = expected(n, spec_rules)
            assert np.array_equal(b.values(), want)
            ranked_equal(corpus, b, want)
            empty = F.Matcher.from_query("", Config(sort=SortStrategy.IndexAsc))
            x, _ = empty.match_list_ranked_array(corpus, b, 100)
            ref = corpus.boost(want)
            y, _ = empty.match_list_ranked_array(corpus, ref, 100)
            assert np.array_equal(x, y)
            ref.close()
            empty.close()
    finally:
        for h in (a, b):
            h.close()
        corpus.close()


@pytest.mark.parametrize("q", [1, 2, 7, 64, 300])
@pytest.mark.parametrize("n", [0, 1025, 100_000])
def test_batch_equals_single(n, q):
    rng = np.random.default_rng(n * 7 + q)
    corpus = new_corpus(n, n + 1)
    vals = attr_values(n, rng) + [rng.integers(0, 5, n).astype(np.int64), rng.integers(0, 3, n).astype(np.int64)]
    attrs = [corpus.attr(v) for v in vals]   # 5 distinct attributes: more than are staged
    shared = corpus.boost(rng.integers(-100, 100, n).astype(np.int16))
    got = [corpus.boost(rng.integers(-10, 10, n).astype(np.int16)) for _ in range(q)]
    twins = [corpus.boost(x.values()) for x in got]
    try:
        rules = [random_rules(attrs, vals, n, rng, 0 if j % 5 == 4 else None)[0] for j in range(q)]
        bases = [(None, shared, "self")[j % 3] for j in range(q)]
        F.boost_where_batch(got, rules, [g if bs == "self" else bs for g, bs in zip(got, bases)])
        for t, r, bs in zip(twins, rules, bases):
            t.where(*r, base=t if bs == "self" else bs)
        for j in range(q):
            assert np.array_equal(got[j].values(), twins[j].values()), (n, q, j)
        if n:
            ms = [F.Matcher(BATCH_NEEDLES[j % len(BATCH_NEEDLES)], Config(max_typos=0, sort=SortStrategy(j % 4))) for j in range(min(q, 40))]
            a = F.match_list_batch(ms, corpus, 10, boosts=got[: len(ms)])
            b = F.match_list_batch(ms, corpus, 10, boosts=[corpus.boost(t.values()) for t in twins[: len(ms)]])
            for x, y in zip(a, b):
                assert np.array_equal(x, y)
            for m in ms:
                m.close()
        # all with one staged-attribute set and no bases
        F.boost_where_batch(got, [[attrs[0].between(0, 500_000).add(j)] for j in range(q)])
        for j in range(q):
            assert np.array_equal(got[j].values(), expected(n, [(spec(full(vals[0], n), 0, 500_000), j)]))
    finally:
        for h in attrs + got + twins + [shared]:
            h.close()
        corpus.close()


def _lib():
    L = F.lib()
    L.frz_debug_device_bytes_peak.restype = C.c_uint64
    L.frz_debug_device_bytes_peak.argtypes = [C.c_int]
    return L


def test_refill_allocates_nothing():
    n = 300_000
    rng = np.random.default_rng(4)
    corpus = new_corpus(n, 4)
    vals = attr_values(n, rng)
    attrs = [corpus.attr(v) for v in vals]
    q = 64
    boosts = [corpus.boost() for _ in range(q)]
    rules = [random_rules(attrs, vals, n, rng)[0] for _ in range(q)]
    F.boost_where_batch(boosts, rules)
    boosts[0].where(*rules[1])
    L = _lib()
    L.frz_debug_device_bytes_peak(1)
    F.boost_where_batch(boosts, rules, boosts)
    boosts[0].where(*rules[1], base=boosts[0])
    peak = L.frz_debug_device_bytes_peak(0)
    F.boost_where_batch(boosts, rules, boosts)
    boosts[0].where(*rules[1], base=boosts[0])
    assert L.frz_debug_device_bytes_peak(0) == peak   # a steady-state refill allocates nothing
    for h in boosts + attrs:
        h.close()
    corpus.close()


def test_refused_calls_leave_every_boost():
    c1, c2 = new_corpus(3000, 5), new_corpus(100, 6)
    a1, a2 = c1.attr(np.arange(3000)), c2.attr(np.arange(100))
    bs = [c1.boost(np.arange(3000) % 7), c1.boost([5]), c1.boost()]
    bs[2].where(a1.between(0, 99).add(3))
    other = c2.boost([4])
    before = [x.values() for x in bs]
    refusals = [
        (lambda: bs[0].where(a2.between(0, 9).add(1)), "the attribute of rule 0 was made on another corpus"),
        (lambda: bs[0].where(base=other), "the base boost was made on another corpus"),
        (lambda: bs[0].where(*[a1.between(0, 9).add(1)] * 9), "9 rules"),
        (lambda: bs[0].where(a1.between(0, 9).add(65536)), "rule 0 adds 65536"),
        (lambda: bs[0].where(a1.isin([1, NULL]).add(1)), "set value 1 of rule 0 is FRZ_ATTR_NULL"),
        (lambda: F.boost_where_batch(bs, [[a1.between(0, 9).add(1)], [a2.between(0, 9).add(1)], []]),
         "query 1: the attribute of rule 0 was made on another corpus"),
        (lambda: F.boost_where_batch(bs + [other], [[], [], [], []]), "query 3: the boost was made on another corpus"),
        (lambda: F.boost_where_batch([bs[0], bs[1], bs[0]], [[], [], []]), "query 2: the boost is also query 0's"),
        (lambda: F.boost_where_batch(bs, [[], [], []], [bs[1], None, None]), "query 0: the base is query 1's boost"),
        (lambda: F.boost_where_batch(bs, [[], [], [a1.between(0, 1).add(-65536)]]), "query 2: rule 0 adds -65536"),
        (lambda: F.boost_where_batch(bs, [[a1.isin(np.arange(4097)).add(1)], [], []]), "query 0: more than 4096 set values"),
    ]
    for call, msg in refusals:
        with pytest.raises(F.FrizbeeError, match=msg):
            call()
        for x, want in zip(bs, before):   # a refused call leaves every boost as it was
            assert np.array_equal(x.values(), want), msg
    with pytest.raises(ValueError):
        F.boost_where_batch(bs, [[], []])
    assert F.boost_where_batch([], []) == []
    for h in bs + [other, a1, a2, c1, c2]:
        h.close()
